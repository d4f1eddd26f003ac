"""Sync committee contributions on the CPU oracle (TEST INFRASTRUCTURE): what b2_sync_contribution_and_proof_intake computes, restated over
oracle.bls_sig and oracle/ssz.py.

Restated from the upstream Altair consensus specs, as recalled, not copied:
  * validator spec: the containers SyncCommitteeContribution, ContributionAndProof, SignedContributionAndProof and
    SyncAggregatorSelectionData; is_sync_committee_aggregator (bytes_to_uint64(hash(selection_proof)[0:8]) modulo max(1, subcommittee size
    // TARGET_AGGREGATORS_PER_SYNC_SUBCOMMITTEE) is zero); process_sync_committee_contributions (the aggregate's bits from the
    contributions' rows, bls.Aggregate of their signatures).
  * p2p, topic sync_committee_contribution_and_proof: IGNORE another slot; REJECT subcommittee_index >= SYNC_COMMITTEE_SUBNET_COUNT, no
    participant, a selection proof that does not select an aggregator, an aggregator outside the subcommittee; IGNORE when a contribution of
    the same root and subcommittee with a superset of the bits was already seen, or when the aggregator already had one accepted for the
    subcommittee; REJECT a bad selection proof, a bad outer signature, and a contribution signature that fails FastAggregateVerify over the
    subcommittee keys of its set bits.
The committee is given as position_validator (the registry index of each position), as the engine takes it; status numbers and the `best`
choice (most bits, ties to the smaller list index) are the engine's (include/b200pos.h).
"""
from collections import namedtuple

from oracle import bls_sig as B
from oracle.bls12_381 import R
from oracle.ssz import compute_signing_root_from_object_root, merkleize, sha256, uint_chunk

from sync_messages_oracle import SyncCommitteeContribution, pack, process_sync_committee_contributions
from sync_oracle import G2_POINT_AT_INFINITY

SUBNET_COUNT = 4
FIXED = 344
NONE = 0xFFFFFFFF
(ACCEPT, MALFORMED, OTHER_SLOT, BAD_SUBNET, NO_BITS, NOT_AGGREGATOR, BAD_AGGREGATOR, NOT_IN_SUBNET, COVERED, SEEN_AGGREGATOR, BAD_PROOF,
 BAD_SIGNATURE, BAD_CONTRIBUTION) = range(13)

# status per item, root_id per item (NONE: not accepted), roots by first accepted occurrence, best[root id][subnet] (NONE: none),
# aggregates [SyncAggregate per root id]
Result = namedtuple("Result", "status root_id roots best aggregates")


def encode(aggregator: int, slot: int, root: bytes, subnet: int, bits, signature: bytes, proof: bytes, outer: bytes) -> bytes:
    """SignedContributionAndProof's SSZ bytes; bits is the Bitvector as bools"""
    return (int(aggregator).to_bytes(8, "little") + int(slot).to_bytes(8, "little") + bytes(root) + int(subnet).to_bytes(8, "little")
            + pack(bits) + bytes(signature) + bytes(proof) + bytes(outer))


def decode(w: bytes, sb: int):
    """-> (aggregator, slot, root, subnet, Bitvector bytes, signature, proof, outer)"""
    u = lambda o: int.from_bytes(w[o:o + 8], "little")      # noqa: E731
    return (u(0), u(8), bytes(w[16:48]), u(48), bytes(w[56:56 + sb]), bytes(w[56 + sb:152 + sb]), bytes(w[152 + sb:248 + sb]),
            bytes(w[248 + sb:344 + sb]))


def bitvector_root(row: bytes) -> bytes:
    """hash_tree_root(Bitvector[n]) of its packed bytes: 32-byte chunks, no length mix-in"""
    return merkleize([row[i:i + 32].ljust(32, b"\0") for i in range(0, max(len(row), 1), 32)])


def sig_root(sig: bytes) -> bytes:
    return merkleize([sig[0:32], sig[32:64], sig[64:96]])


def contribution_root(slot, root, subnet, row: bytes, signature) -> bytes:
    return merkleize([uint_chunk(slot), bytes(root), uint_chunk(subnet), bitvector_root(row), sig_root(signature)])


def contribution_and_proof_root(aggregator, slot, root, subnet, row: bytes, signature, proof) -> bytes:
    return merkleize([uint_chunk(aggregator), contribution_root(slot, root, subnet, row, signature), sig_root(proof)])


def selection_data_root(slot, subnet) -> bytes:
    return merkleize([uint_chunk(slot), uint_chunk(subnet)])


def signing_root(object_root: bytes, domain32: bytes) -> bytes:
    return compute_signing_root_from_object_root(object_root, domain32)


def is_aggregator(proof: bytes, sub: int, target: int) -> bool:
    return int.from_bytes(sha256(bytes(proof))[0:8], "little") % max(1, sub // target) == 0


def _bits(row: bytes, sub: int):
    return [bool(row[i >> 3] >> (i & 7) & 1) for i in range(sub)]


def validate(wires, position_validator, n_validators, pubkey_of, current_slot, domains96, target=16, count=SUBNET_COUNT, verify=None,
             fast_verify=None, secret_key=None, closed_form=False):
    """verify(item, pubkey, message, signature, which) with which 0 (selection proof) or 1 (outer signature) defaults to bls.Verify;
    fast_verify(item, pubkeys, message, signature) to bls.FastAggregateVerify.  With secret_key(validator) given, each aggregate's
    signature is computed in closed form, Sign(sum of the secret keys of its set positions, a validator at k positions k times, message):
    the accepted contributions must then be honest ones.  With closed_form as well, it is left as the pair (sum mod r, signing root) for
    the caller to sign in one batch (sync_messages_oracle.sign_closed_form)."""
    verify = verify or (lambda a, pk, m, s, which: B.Verify(pk, m, s))
    fast_verify = fast_verify or (lambda a, pks, m, s: B.FastAggregateVerify(pks, m, s))
    dom_sync, dom_sel, dom_cap = domains96[0:32], domains96[32:64], domains96[64:96]
    size = len(position_validator)
    sub = size // count
    sb = (sub + 7) // 8
    status, acc = [], []      # acc: (item, root, subnet, aggregator, bits as an int) of the accepted items
    for a, w in enumerate(wires):
        w = bytes(w)
        if len(w) != FIXED + sb or (sub & 7 and w[56 + sb - 1] >> (sub & 7)):
            status.append(MALFORMED)
            continue
        g, slot, root, s, row, sig, proof, outer = decode(w, sb)
        bits = _bits(row, sub)
        mask = int.from_bytes(row, "little")
        if slot != current_slot:
            st = OTHER_SLOT
        elif s >= count:
            st = BAD_SUBNET
        elif not any(bits):
            st = NO_BITS
        elif not is_aggregator(proof, sub, target):
            st = NOT_AGGREGATOR
        elif g >= n_validators:
            st = BAD_AGGREGATOR
        elif g not in position_validator[s * sub:(s + 1) * sub]:
            st = NOT_IN_SUBNET
        elif any(r == root and t == s and mask & ~b == 0 for _, r, t, _, b in acc):
            st = COVERED
        elif any(h == g and t == s for _, _, t, h, _ in acc):
            st = SEEN_AGGREGATOR
        elif not verify(a, pubkey_of(g), signing_root(selection_data_root(slot, s), dom_sel), proof, 0):
            st = BAD_PROOF
        elif not verify(a, pubkey_of(g), signing_root(contribution_and_proof_root(g, slot, root, s, row, sig, proof), dom_cap), outer, 1):
            st = BAD_SIGNATURE
        elif not fast_verify(a, [pubkey_of(position_validator[s * sub + i]) for i in range(sub) if bits[i]], signing_root(root, dom_sync), sig):
            st = BAD_CONTRIBUTION
        else:
            st = ACCEPT
            acc.append((a, root, s, g, mask))
        status.append(st)
    roots, root_id = [], [NONE] * len(wires)
    for a, root, _, _, _ in acc:
        if root not in roots:
            roots.append(root)
        root_id[a] = roots.index(root)
    best = [[NONE] * count for _ in roots]
    for a, root, s, _, mask in acc:
        r, b = roots.index(root), best[roots.index(root)][s]
        if b == NONE or bin(mask).count("1") > bin(int.from_bytes(decode(bytes(wires[b]), sb)[4], "little")).count("1"):
            best[r][s] = a
    aggregates = []
    for r, root in enumerate(roots):
        present = []
        for s in range(count):
            if best[r][s] != NONE:
                g, slot, _, _, row, sig, _, _ = decode(bytes(wires[best[r][s]]), sb)
                present.append(SyncCommitteeContribution(slot, root, s, _bits(row, sub), sig))
        agg = process_sync_committee_contributions(present, size, count, aggregate=secret_key is None)
        if secret_key is not None:
            k = sum(secret_key(position_validator[p]) for p, on in enumerate(agg.sync_committee_bits) if on) % R
            msg = signing_root(root, dom_sync)
            agg.sync_committee_signature = (k, msg) if closed_form else B.Sign(k, msg) if k else G2_POINT_AT_INFINITY
        aggregates.append(agg)
    return Result(status, root_id, roots, best, aggregates)


class Signer:
    """Honest and corrupted items over a committee of scenarios' keys (secret key scenarios.secret_key(v)), or of secret_key(v)"""

    def __init__(self, position_validator, domains96, slot, count=SUBNET_COUNT, secret_key=None):
        import scenarios
        self.pv, self.dom, self.slot, self.count = list(position_validator), bytes(domains96), slot, count
        self.sub = len(self.pv) // count
        self.sk = secret_key or scenarios.secret_key

    def proof(self, v, s, sk=None, slot=None):
        slot = self.slot if slot is None else slot
        return B.Sign(self.sk(v) if sk is None else sk, signing_root(selection_data_root(slot, s), self.dom[32:64]))

    def contribution_signature(self, s, bits, root, delta=0):
        """Sign(the sum of the secret keys of the set positions (a validator at k positions k times) + delta, signing root)"""
        k = sum(self.sk(self.pv[s * self.sub + i]) for i, b in enumerate(bits) if b) + delta
        return B.Sign(k % R, signing_root(root, self.dom[0:32])) if k % R else bytes([0xC0]) + bytes(95)

    def item(self, v, s, root, bits, slot=None, proof=None, bad_outer=False, bad_sig=False, subnet_field=None):
        slot = self.slot if slot is None else slot
        proof = self.proof(v, s, slot=slot) if proof is None else proof
        sig = self.contribution_signature(s, bits, root, 1 if bad_sig else 0)
        s_field = s if subnet_field is None else subnet_field
        row = pack(bits)
        cap = signing_root(contribution_and_proof_root(v, slot, root, s_field, row, sig, proof), self.dom[64:96])
        outer = B.Sign(self.sk(v) + (1 if bad_outer else 0), cap)
        return encode(v, slot, root, s_field, bits, sig, proof, outer)

    def bad_proof(self, v, s, target, want_aggregator=True):
        """a selection proof of v's that is not its own signature and whose hash does (or does not) select an aggregator"""
        for k in range(1, 200):
            p = self.proof(v, s, sk=self.sk(v) + k)
            if is_aggregator(p, self.sub, target) == want_aggregator:
                return p
        raise AssertionError("no proof found")


def expect_arrays(r: Result, count=SUBNET_COUNT, size=None):
    """the oracle's Result as the engine's trimmed arrays: status, root_id, roots, best, agg_bits, agg_sigs"""
    import numpy as np
    k = len(r.roots)
    ab = (size + 7) // 8
    bits, sigs = np.zeros((k, ab), np.uint8), np.zeros((k, 96), np.uint8)
    for j, a in enumerate(r.aggregates):
        bits[j] = np.frombuffer(pack(a.sync_committee_bits), np.uint8)
        sigs[j] = np.frombuffer(a.sync_committee_signature, np.uint8)
    roots = np.frombuffer(b"".join(r.roots), np.uint8).reshape(k, 32) if k else np.zeros((0, 32), np.uint8)
    best = np.array(r.best, np.uint32).reshape(k, count)
    return (np.array(r.status, np.int32), np.array(r.root_id, np.uint32), roots, best, bits, sigs)


def with_aggregators(position_validator, n_validators, signer_of, target, need):
    """position_validator with, for each subnet s in need, need[s] validators whose own selection proof selects them placed at the
    subnet's first positions (signer_of(pv) -> Signer)"""
    pv = list(position_validator)
    sg = signer_of(pv)
    for s, k in need.items():
        found = [v for v in range(n_validators) if is_aggregator(sg.proof(v, s), sg.sub, target)][:k]
        assert len(found) == k
        pv[s * sg.sub:s * sg.sub + k] = found
    return pv


def scenario(sg: Signer, roots, target, n_validators):
    """(wires, expected statuses) reaching every status 0-12 at a target below the subcommittee size (subnets 1 and 2 must each have two
    aggregators at their first positions and subnet 3 one, as with_aggregators(..., {1: 2, 2: 2, 3: 1}) places them; a third root adds an
    accepted item on subnet 3): list-order cases -- a bad selection proof before the aggregator's accepted item, a covered
    subset, an equal-bits duplicate, the same aggregator on a second root, a subset accepted after two rejected supersets, equal-size
    contributions of two aggregators on one (root, subnet) -- and every rejection before the signatures"""
    sub, pv = sg.sub, sg.pv
    r0, r1 = roots[0], roots[1]
    a1, a3, b1, b2 = pv[sub], pv[sub + 1], pv[2 * sub], pv[2 * sub + 1]
    a2 = pv[sub + 2]
    on = lambda *ix: [i in ix for i in range(sub)]      # noqa: E731
    out = []

    def add(w, st):
        out.append((w, st))

    add(sg.item(a1, 1, r0, on(0, 1, 2), proof=sg.bad_proof(a1, 1, target)), BAD_PROOF)      # does not shadow a1's next item
    add(sg.item(a1, 1, r0, on(0, 1, 2)), ACCEPT)
    add(sg.item(a1, 1, r0, on(1)), COVERED)
    add(sg.item(a3, 1, r0, on(0, 1, 2)), COVERED)                                              # equal bits
    add(sg.item(a1, 1, r1, on(0, 1, 2, 3)), SEEN_AGGREGATOR)                                    # a second root
    add(sg.item(a3, 1, r1, on(0, 1, 2, 3, 4, 5), bad_outer=True), BAD_SIGNATURE)
    add(sg.item(a3, 1, r1, on(0, 1, 2, 3, 4, 5), bad_sig=True), BAD_CONTRIBUTION)
    add(sg.item(a3, 1, r1, on(2, 3)), ACCEPT)                                                  # a subset of two rejected supersets
    add(sg.item(b1, 2, r1, on(4, 5)), ACCEPT)
    add(sg.item(b2, 2, r1, on(6, 7)), ACCEPT)                                                  # ties with b1's: b1 stays best
    add(sg.item(b2, 2, r1, on(0, 1, 2)), SEEN_AGGREGATOR)
    add(sg.item(b1, 2, r0, on(0, 1, 2, 3, 4, 5, 6, 7)), SEEN_AGGREGATOR)
    if len(roots) > 2:
        add(sg.item(pv[3 * sub], 3, roots[2], on(0, 1)), ACCEPT)
    add(sg.item(a2, 1, r0, on(3), proof=sg.bad_proof(a2, 1, target, False)) if target < sub else sg.item(a2, 1, r0, on(3)),
        NOT_AGGREGATOR if target < sub else ACCEPT)
    add(sg.item(a1, 1, r0, on(0), slot=sg.slot + 1), OTHER_SLOT)
    add(sg.item(a1, 1, r0, on(0), subnet_field=sg.count), BAD_SUBNET)
    add(sg.item(a1, 1, r0, on()), NO_BITS)
    add(sg.item(n_validators, 1, r0, on(0), proof=sg.bad_proof(a1, 1, target)), BAD_AGGREGATOR)
    outsider = next(v for v in range(n_validators) if v not in pv[sub:2 * sub])
    add(sg.item(outsider, 1, r0, on(0), proof=sg.bad_proof(outsider, 1, target)), NOT_IN_SUBNET)
    add(sg.item(a1, 1, r0, on(0))[:-1], MALFORMED)
    return [w for w, _ in out], [st for _, st in out]
