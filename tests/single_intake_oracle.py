"""Host oracle of the SingleAttestation intake (include/b200pos.h, b2_single_attestation_intake): one epoch of Electra's unaggregated
attestations (EIP-7549, the beacon_attestation_{subnet_id} topic) on the wire, checked item by item in list order as the upstream Electra
p2p conditions and validate_on_attestation (upstream fork-choice spec v1.2.0, :963-979) require against a block store, one kept per
attester, grouped by AttestationData into the vote form's inputs.

single_intake_plain restates the contract over oracle.spec containers, a block dict (intake_oracle.block_store) and oracle.spec's
get_ancestor and hash_tree_root_attestation_data.  as_phase0 rewrites an item as the phase 0 Attestation the phase 0 intake reads."""
import types

import numpy as np

from oracle.spec import Spec, hash_tree_root_attestation_data
from oracle.ssz import compute_signing_root_from_object_root

import intake_oracle as IO

SIZE = 240
NONE = 0xFFFFFFFF


def compute_subnet_for_attestation(committees_per_slot, slot, committee_index, slots_per_epoch, subnet_count):
    """upstream phase 0 validator spec, with Electra's committee_index in data.index's place"""
    slots_since_epoch_start = slot % slots_per_epoch
    committees_since_epoch_start = committees_per_slot * slots_since_epoch_start
    return (committees_since_epoch_start + committee_index) % subnet_count


def encode(committee_index, attester_index, data128: bytes, signature: bytes) -> bytes:
    return int(committee_index).to_bytes(8, "little") + int(attester_index).to_bytes(8, "little") + bytes(data128) + bytes(signature)


def single_intake_plain(wires, subnets, members, off, epoch, current_slot, domain, committees_per_slot, slots_per_epoch, blocks, ids,
                        subnet_count=64):
    """wires: one encoding per item (list order); subnets: the subnet each arrived on; members / off: the committees; blocks / ids:
    intake_oracle.block_store's.  Every vote row, not only the first max_votes."""
    store = types.SimpleNamespace(blocks=blocks)
    start = epoch * slots_per_epoch
    status, kept = [], {}
    for i, w in enumerate(wires):
        w = bytes(w)
        st = 0
        if len(w) != SIZE:
            st = 1
        else:
            committee_index, attester = int.from_bytes(w[0:8], "little"), int.from_bytes(w[8:16], "little")
            data = IO.data_from_bytes(w[16:144])
            if data.index != 0:
                st = 2
            elif committee_index >= committees_per_slot:
                st = 3
            elif not start <= data.slot < start + slots_per_epoch:
                st = 4
            elif compute_subnet_for_attestation(committees_per_slot, data.slot, committee_index, slots_per_epoch, subnet_count) != int(subnets[i]):
                st = 5
            elif data.target.epoch != epoch:
                st = 6
            elif current_slot < data.slot + 1:
                st = 7
            else:
                c = (data.slot - start) * committees_per_slot + committee_index
                committee = [int(x) for x in members[int(off[c]):int(off[c + 1])]]
                if attester not in committee:
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
                    p = committee.index(attester)
                    if anc != data.target.root:
                        st = 12
                    elif (c, p) in kept:
                        st = 13
                    else:
                        kept[(c, p)] = (w[16:144], w[144:240], data)
        status.append(st)
    n_c, n_sig = len(off) - 1, int(off[-1])
    vote = np.full(n_sig, NONE, dtype=np.uint32)
    sigs = np.zeros((n_sig, 96), dtype=np.uint8)
    vote_off, rows = [0], []
    for c in range(n_c):
        groups = {}
        for p in range(int(off[c + 1]) - int(off[c])):
            if (c, p) in kept:
                groups.setdefault(kept[(c, p)][0], []).append(p)      # positions ascend: a group's first is its smallest
        for d in sorted(groups, key=lambda d: groups[d][0]):
            v = len(rows)
            data = kept[(c, groups[d][0])][2]
            msg = compute_signing_root_from_object_root(hash_tree_root_attestation_data(data), domain)
            rows.append((d, msg, data.source.epoch, data.target.epoch, ids[data.beacon_block_root]))
            for p in groups[d]:
                vote[int(off[c]) + p] = v
                sigs[int(off[c]) + p] = np.frombuffer(kept[(c, p)][1], dtype=np.uint8)
        if not groups:
            rows.append((bytes(128), bytes(32), 0, 0, 0))
        vote_off.append(len(rows))
    return IO._result(np.array(status, dtype=np.int32), vote, np.array(vote_off, dtype=np.int64), sigs, rows)


def as_phase0(w: bytes, members, off, committees_per_slot, slots_per_epoch, epoch):
    """The phase 0 Attestation of a kept item: data.index = committee_index and one bit at the attester's position"""
    w = bytes(w)
    ci, who = int.from_bytes(w[0:8], "little"), int.from_bytes(w[8:16], "little")
    d = bytearray(w[16:144])
    slot = int.from_bytes(d[0:8], "little")
    c = (slot - epoch * slots_per_epoch) * committees_per_slot + ci
    committee = [int(x) for x in members[int(off[c]):int(off[c + 1])]]
    d[8:16] = ci.to_bytes(8, "little")
    return IO.encode([m == who for m in committee], bytes(d), w[144:240])


def subnets_of(wires, committees_per_slot, slots_per_epoch, subnet_count=64):
    """the subnet each well-formed item belongs on (0 for an item too short to name one)"""
    out = []
    for w in wires:
        if len(w) < 24:
            out.append(0)
            continue
        ci, slot = int.from_bytes(w[0:8], "little"), int.from_bytes(w[16:24], "little")
        out.append(compute_subnet_for_attestation(committees_per_slot, slot, ci, slots_per_epoch, subnet_count) & 0xFFFFFFFF)
    return np.array(out, dtype=np.uint32)


# ------------------------------------------------------------------------------------------ test epochs
def random_epoch(rng, epoch, spe, cps, members, off, tree, n_validators, corrupt=0.3, dup=0.1, heads_per_committee=2, subnet_count=64):
    """(wires, subnets) of one epoch: every member of every committee attests once to one of a few heads of its committee, in random
    order; a share `corrupt` is broken in one way (statuses 1-12; the subnet of status 5 is in `subnets`); then, for a share `dup`, a
    second item of the same attester is appended, with equal or other data."""
    parent, slot, roots = tree
    start = epoch * spe
    wires, subnets = [], []
    sig = lambda: rng.integers(0, 256, size=96, dtype=np.uint8).tobytes()      # noqa: E731
    for c in range(spe * cps):
        s, ci = start + c // cps, c % cps
        ok = [b for b in range(len(parent)) if int(slot[b]) <= s and IO.ancestor(parent, slot, b, start) is not None] or [0]
        heads = []
        for _ in range(heads_per_committee):
            h = ok[int(rng.integers(0, len(ok)))]
            t = IO.ancestor(parent, slot, h, start)
            heads.append(IO.data128(s, 0, bytes(roots[h]), epoch - 1 if epoch else 0, bytes(roots[0]), epoch, bytes(roots[0 if t is None else t])))
        committee = members[int(off[c]):int(off[c + 1])]
        for v in committee.tolist():
            d, who, cidx = bytearray(heads[int(rng.integers(0, len(heads)))]), int(v), ci
            net = compute_subnet_for_attestation(cps, s, ci, spe, subnet_count)
            kind = int(rng.integers(0, 12)) if rng.random() < corrupt else -1
            if kind == 1:
                d[8:16] = (1).to_bytes(8, "little")                            # data.index != 0
            elif kind == 2:
                cidx = cps + int(rng.integers(0, 3))                            # committee index out of range
            elif kind == 3:
                d[0:8] = (start + spe + int(rng.integers(0, 3))).to_bytes(8, "little")      # slot outside the epoch
            elif kind == 4:
                net = (net + 1 + int(rng.integers(0, subnet_count - 1))) % subnet_count      # another subnet
            elif kind == 5:
                d[88:96] = (epoch + 1).to_bytes(8, "little")                    # target epoch
            elif kind == 6:
                who = n_validators + int(rng.integers(0, 5))                    # not a member
            elif kind == 7:
                d[16:48] = bytes([0xAB] * 32)                                   # unknown head
            elif kind == 8:
                d[96:128] = bytes([0xCD] * 32)                                  # unknown target
            elif kind == 9:
                d[16:48] = bytes(roots[int(np.argmax(slot))])                   # the newest block: usually newer than data.slot
            elif kind == 10:
                d[96:128] = bytes(roots[int(rng.integers(0, len(parent)))])    # a known block, usually not the ancestor
            w = encode(cidx, who, bytes(d), sig())
            if kind == 0:
                w = w[:SIZE - 1 - int(rng.integers(0, 8))] if rng.random() < 0.5 else w + bytes(1)      # not 240 bytes
            elif kind == 11:
                who = int(members[int(off[(c + 1) % (spe * cps)])])             # a member of another committee
                w = encode(cidx, who, bytes(d), sig())
            wires.append(w)
            subnets.append(net)
    order = rng.permutation(len(wires))
    wires, subnets = [wires[i] for i in order], [subnets[i] for i in order]
    for i in np.nonzero(rng.random(len(wires)) < dup)[0].tolist():
        w = bytearray(wires[i])
        if len(w) == SIZE and rng.random() < 0.5:
            w[16 + 56] ^= 1                                                     # other data (source root), the same attester
        w[-96:] = sig()
        wires.append(bytes(w))
        subnets.append(subnets[i])
    return wires, np.array(subnets, dtype=np.uint32)
