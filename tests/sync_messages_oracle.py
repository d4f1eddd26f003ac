"""Sync committee messages on the CPU oracle (TEST INFRASTRUCTURE): what b2_sync_committee_messages computes, restated over oracle.bls_sig
and tests/sync_oracle.py.

The reference names the container, SyncCommitteeMessage (pos-evolution.md:548-557).  The rest is restated from the upstream Altair
consensus specs, as recalled, not copied:
  * p2p, topic sync_committee_{subnet_id}: IGNORE a message of another slot; REJECT a subnet_id that is not in
    compute_subnets_for_sync_committee(state, validator_index); IGNORE when a message of the same (validator_index, slot, subnet_id) was
    already accepted; REJECT a bad signature over compute_signing_root(beacon_block_root, get_domain(DOMAIN_SYNC_COMMITTEE, epoch of slot)).
  * validator spec: the SyncCommitteeContribution of a subnet sets bit i for the member at position subnet * subcommittee size + i that
    signed, with the signatures summed; process_sync_committee_contributions sets the aggregate's bits from the contributions' rows and
    signs with bls.Aggregate of their signatures.
The committee is given as position_validator (the registry index of each position), as the engine takes it; status numbers are the
engine's (include/b200pos.h).
"""
import hashlib
from collections import namedtuple
from dataclasses import dataclass
from typing import List

from oracle import bls_sig as B
from oracle.bls12_381 import R

from sync_oracle import G2_POINT_AT_INFINITY, SyncAggregate

SUBNET_COUNT = 4
WIRE = 144
NONE = 0xFFFFFFFF
ACCEPT, MALFORMED, OTHER_SLOT, BAD_VALIDATOR, BAD_SUBNET, SEEN, BAD_SIGNATURE = range(7)


@dataclass
class SyncCommitteeContribution:
    slot: int
    beacon_block_root: bytes
    subcommittee_index: int
    aggregation_bits: List[bool]
    signature: bytes


# status per item, root_id per item (NONE: not accepted), roots in first-occurrence order, contributions {(root id, subnet): contribution}
# (present ones only), aggregates [SyncAggregate per root id]
Result = namedtuple("Result", "status root_id roots contributions aggregates")


def encode(slot: int, root: bytes, validator_index: int, signature: bytes) -> bytes:
    return int(slot).to_bytes(8, "little") + bytes(root) + int(validator_index).to_bytes(8, "little") + bytes(signature)


def signing_root(root: bytes, domain32: bytes) -> bytes:
    """compute_signing_root(beacon_block_root, domain): hash_tree_root(SigningData) = sha256 of the two chunks"""
    return hashlib.sha256(bytes(root) + bytes(domain32)).digest()


def subnets_of(position_validator, validator_index: int, count: int = SUBNET_COUNT):
    """compute_subnets_for_sync_committee over registry indices"""
    sub = len(position_validator) // count
    return {p // sub for p, v in enumerate(position_validator) if v == validator_index}


def validate(wires, subnets, position_validator, n_validators, pubkey_of, current_slot, domain32, count=SUBNET_COUNT, verify=None,
             secret_key=None, closed_form=False):
    """verify(item, pubkey, message, signature) defaults to bls.Verify.  With secret_key(validator) given, every sum of accepted signatures
    is computed in closed form, Sign(sum of the signers' secret keys, message): the accepted signatures must then be honest ones.  With
    closed_form as well, each such signature is left as its pair (sum of the secret keys mod r, signing root), for the caller to sign in one
    batch (sign_closed_form)."""
    verify = verify or (lambda a, pk, msg, sig: B.Verify(pk, msg, sig))
    size = len(position_validator)
    sub = size // count
    status, seen, acc = [], set(), {}      # acc[(validator, subnet)] = accepted item
    for a, w in enumerate(wires):
        w = bytes(w)
        if len(w) != WIRE:
            status.append(MALFORMED)
            continue
        slot, root = int.from_bytes(w[0:8], "little"), w[8:40]
        v, sig, s = int.from_bytes(w[40:48], "little"), w[48:144], int(subnets[a])
        if slot != current_slot:
            st = OTHER_SLOT
        elif v >= n_validators:
            st = BAD_VALIDATOR
        elif s not in subnets_of(position_validator, v, count):
            st = BAD_SUBNET
        elif (v, s) in seen:
            st = SEEN
        elif not verify(a, pubkey_of(v), signing_root(root, domain32), sig):
            st = BAD_SIGNATURE
        else:
            st = ACCEPT
            seen.add((v, s))
            acc[(v, s)] = a
        status.append(st)
    roots, root_id = [], [NONE] * len(wires)
    for a, st in enumerate(status):
        if st == ACCEPT:
            r = bytes(wires[a])[8:40]
            if r not in roots:
                roots.append(r)
            root_id[a] = roots.index(r)

    def sig_sum(items, signers, msg):
        if secret_key is not None:
            k = sum(secret_key(v) for v in signers) % R
            return (k, msg) if closed_form else B.Sign(k, msg)
        return B.Aggregate([bytes(wires[a])[48:144] for a in items])

    contributions, aggregates = {}, []
    for r, root in enumerate(roots):
        msg = signing_root(root, domain32)
        for s in range(count):
            bits, items, signers = [], [], []
            for i in range(sub):
                v = position_validator[s * sub + i]
                a = acc.get((v, s))
                on = a is not None and root_id[a] == r
                bits.append(on)
                if on:
                    items.append(a)
                    signers.append(v)
            if items:
                contributions[(r, s)] = SyncCommitteeContribution(current_slot, root, s, bits, sig_sum(items, signers, msg))
        present = [contributions[(r, s)] for s in range(count) if (r, s) in contributions]
        agg = process_sync_committee_contributions(present, size, count, aggregate=secret_key is None)
        if secret_key is not None:      # the closed form of the same sum
            agg.sync_committee_signature = sig_sum(None, [position_validator[p] for p, b in enumerate(agg.sync_committee_bits) if b], msg)
        aggregates.append(agg)
    return Result(status, root_id, roots, contributions, aggregates)


def closed_form_pairs(r):
    """every (secret key, message) pair of a closed-form Result, in a fixed order (contributions by key, then aggregates)"""
    out = [c.signature for _, c in sorted(r.contributions.items())] if hasattr(r, "contributions") else []
    return out + [a.sync_committee_signature for a in r.aggregates]


def sign_closed_form(r, sign):
    """the Result with each (secret key, message) pair replaced by its signature: sign(keys, messages) -> signatures, one batch (a zero
    key sums to the point at infinity)"""
    pairs = [p for p in closed_form_pairs(r) if isinstance(p, tuple)]
    live = [p for p in pairs if p[0] % R]
    sigs = dict(zip(live, sign([k for k, _ in live], [m for _, m in live]))) if live else {}
    done = lambda p: (sigs[p] if p[0] % R else G2_POINT_AT_INFINITY) if isinstance(p, tuple) else p      # noqa: E731
    if hasattr(r, "contributions"):
        for c in r.contributions.values():
            c.signature = done(c.signature)
    for a in r.aggregates:
        a.sync_committee_signature = done(a.sync_committee_signature)
    return r


def process_sync_committee_contributions(contributions, size, count=SUBNET_COUNT, aggregate=True) -> SyncAggregate:
    """upstream Altair validator spec: the contributions' rows into the aggregate's bits, bls.Aggregate of their signatures (the G2
    infinity encoding when there is none; None without `aggregate`, for a caller that fills in the closed form)"""
    bits, sigs = [False] * size, []
    sub = size // count
    for c in contributions:
        for i, on in enumerate(c.aggregation_bits):
            if on:
                bits[sub * c.subcommittee_index + i] = True
        sigs.append(c.signature)
    if not aggregate:
        return SyncAggregate(bits, None)
    return SyncAggregate(bits, B.Aggregate(sigs) if sigs else G2_POINT_AT_INFINITY)


def pack(bits) -> bytes:
    """a Bitvector's SSZ bytes"""
    out = bytearray((len(bits) + 7) // 8)
    for i, b in enumerate(bits):
        if b:
            out[i >> 3] |= 1 << (i & 7)
    return bytes(out)


def message(v, root, domain, slot, sk=None):
    """v's honest message (secret key scenarios.secret_key(v)), or one signed with `sk`"""
    import scenarios
    sig = B.Sign(scenarios.secret_key(v) if sk is None else sk, signing_root(root, domain))
    return encode(slot, root, v, sig)


def scenario(committee, domain, slot, roots, root_of, n_validators):
    """(wires, subnets, expected statuses) over a minimal committee (8 positions per subnet) of scenarios' keys: every (validator, subnet)
    of the committee once, on roots[root_of(first position)], plus every rejection: a bad signature before the good message of its
    (validator, subnet), duplicates after an accepted message (with a good and a bad signature), another slot, a validator outside the
    registry, a wrong subnet and one >= SUBNET_COUNT, a short encoding"""
    import scenarios
    wires, subnets, expect, sent = [], [], [], set()

    def add(w, s, st):
        wires.append(w)
        subnets.append(s)
        expect.append(st)

    r0 = roots[0]
    v9 = committee[9]
    add(message(v9, roots[root_of(9)], domain, slot, sk=scenarios.secret_key(v9) + 1), 1, BAD_SIGNATURE)
    for p in range(len(committee)):
        v, s = committee[p], p // 8
        if (v, s) in sent:
            continue
        sent.add((v, s))
        add(message(v, roots[root_of(p)], domain, slot), s, ACCEPT)
    add(message(committee[5], r0, domain, slot), 0, SEEN)
    add(message(committee[6], r0, domain, slot, sk=scenarios.secret_key(committee[6]) + 1), 0, SEEN)
    add(message(committee[7], r0, domain, slot + 1), 0, OTHER_SLOT)
    add(encode(slot, r0, n_validators, bytes(96)), 0, BAD_VALIDATOR)
    add(message(committee[8], r0, domain, slot), 0, BAD_SUBNET)
    add(message(committee[8], r0, domain, slot), 4, BAD_SUBNET)
    add(message(committee[0], r0, domain, slot)[:143], 0, MALFORMED)
    return wires, subnets, expect

