"""Array-level host API over the C ABI: one Engine = one b2_ctx = one GPU.

Everything here takes/returns flat numpy arrays (host entry points) or torch CUDA tensors
(`*_dev`, asynchronous on torch's current stream).  The pyspec-signature layer (bls.py, spec.py)
and bench.py are built on it.  No CPU fallback: constructing an Engine without an H100 (sm_90) raises.
"""
import ctypes
from collections import namedtuple

import numpy as np

from . import _lib
from ._lib import B2Error

# Engine.pack_attestations: per pick (in pick order) committee, data id, union bit row, u64 numerator; constituents src[src_off[o] ..
# src_off[o+1]) in pool order; signature (bls.Aggregate of the constituents); cand_status per candidate (0 folded, 1 undecodable)
PackResult = namedtuple("PackResult", "committee data bits numerator src_off src signature cand_status")
# Engine.attestation_intake: status per attestation; the vote form's inputs: vote per member slot, vote_off per committee, signatures in
# committee order, and per vote (max_votes rows) the AttestationData, signing root, source and target epoch and block id
IntakeResult = namedtuple("IntakeResult", "status vote vote_off sigs data128 msgs source_epoch target_epoch block_idx")
# Engine.aggregate_and_proof_intake: per SignedAggregateAndProof its status (0-20), committee, data id, bit row, aggregate signature, attestation
# signing root, target epoch and block id; the member rows (u32[n][8 * bits_stride]) and their offsets item_off (u32[n+1]), the committee
# arrays latest_messages_update / fast_aggregate_verify take with the bit rows
AggregateIntakeResult = namedtuple("AggregateIntakeResult", "status committee data_id bits sigs msgs target_epoch block_idx members item_off")
# Engine.block_attestations: per attestation its status (0-11), participation flag mask and proposer_reward_numerator; per block its status
# (0 applied, 1 invalid, 2 after an invalid block), the list index of its first failing attestation (0xFFFFFFFF: none) and proposer reward;
# the number of blocks applied.  Engine.block_attestations_electra returns the same fields, its statuses 0-13.
BlockAttestationsResult = namedtuple("BlockAttestationsResult", "status flag_mask numerator block_status block_first block_reward n_applied")
# Engine.sync_committee_messages: per message its status (0-6) and root id (0xFFFFFFFF: not accepted); the n_roots distinct roots; per (root,
# subnet) the contribution's bit row, signature and present byte (uint8[n_roots, subnet_count, ...]); per root the SyncAggregate's bit row and
# signature
SyncMessagesResult = namedtuple("SyncMessagesResult", "status root_id roots contrib_bits contrib_sigs contrib_present agg_bits agg_sigs")
# Engine.sync_contribution_and_proof_intake: per SignedContributionAndProof its status (0-12) and root id (0xFFFFFFFF: not accepted); the n_roots
# distinct roots; per (root, subnet) the list index of the best accepted contribution (0xFFFFFFFF: none); per root the SyncAggregate's bit row
# and signature
SyncContributionsResult = namedtuple("SyncContributionsResult", "status root_id roots best agg_bits agg_sigs")


def _c(a, dtype):
    a = np.ascontiguousarray(a, dtype=dtype)
    return a


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p) if a is not None else None


class Engine:
    def __init__(self, device: int = 0):
        self.lib = _lib.load()
        h = ctypes.c_void_p()
        rc = self.lib.b2_init(int(device), ctypes.byref(h))
        if rc != 0:
            raise B2Error(rc, "b2_init(device=%d) failed -- an H100 (sm_90) GPU is required; there is no CPU fallback" % device)
        self.h = h
        self.device = device
        self.n_validators = 0
        self.n_blocks = 0
        self.ssz_loads = 0          # successful ssz_validators_load calls: which tree is on the device

    def close(self):
        if getattr(self, "h", None):
            self.lib.b2_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _ck(self, rc):
        if rc != 0:
            raise B2Error(rc, self.lib.b2_last_error(self.h).decode())

    def sync(self):
        self._ck(self.lib.b2_sync(self.h))

    @property
    def launch_count(self) -> int:
        return int(self.lib.b2_launch_count(self.h))

    # ------------------------------------------------------------------ registry
    def registry_load(self, pubkeys48, effective_balance, flags=None):
        """pubkeys48: uint8[N,48]; effective_balance: uint64[N]; flags: uint8[N] (bit0 active, bit1 slashed).
        Returns uint8[N]: 1 where KeyValidate passed."""
        pk = _c(pubkeys48, np.uint8).reshape(-1, 48)
        n = pk.shape[0]
        eff = _c(effective_balance, np.uint64)
        fl = _c(flags if flags is not None else np.ones(n, dtype=np.uint8), np.uint8)
        assert eff.shape == (n,) and fl.shape == (n,)
        valid = np.zeros(n, dtype=np.uint8)
        self._ck(self.lib.b2_registry_load(self.h, _p(pk), _p(eff), _p(fl), n, _p(valid)))
        self.n_validators = n
        return valid

    def key_validate(self, pubkeys48):
        """bls.KeyValidate for explicit pubkeys (uint8[n,48]) -> uint8[n]; the registry on the device is not touched."""
        pk = _c(pubkeys48, np.uint8).reshape(-1, 48)
        out = np.zeros(pk.shape[0], dtype=np.uint8)
        self._ck(self.lib.b2_key_validate(self.h, _p(pk), pk.shape[0], _p(out)))
        return out

    def registry_update_balances(self, effective_balance, flags):
        eff, fl = _c(effective_balance, np.uint64), _c(flags, np.uint8)
        self._ck(self.lib.b2_registry_update_balances(self.h, _p(eff), _p(fl), eff.shape[0]))

    # ------------------------------------------------------------------ BLS batches
    @staticmethod
    def _batch(members, off, bits):
        members = _c(members, np.uint32)
        off = _c(off, np.uint32)
        bits = _c(bits, np.uint8)
        n_agg = off.shape[0] - 1
        assert bits.ndim == 2 and bits.shape[0] == n_agg
        return members, off, bits, n_agg, bits.shape[1]

    def g1_aggregate(self, members, off, bits):
        members, off, bits, n_agg, stride = self._batch(members, off, bits)
        out = np.zeros((n_agg, 48), dtype=np.uint8)
        status = np.zeros(n_agg, dtype=np.uint8)
        self._ck(self.lib.b2_g1_aggregate(self.h, _p(members), _p(off), _p(bits), stride, n_agg, _p(out), _p(status)))
        return out, status

    def aggregate(self, sigs96, seg_off):
        sigs = _c(sigs96, np.uint8).reshape(-1, 96)
        seg_off = _c(seg_off, np.uint32)
        n_seg = seg_off.shape[0] - 1
        assert int(seg_off[-1]) == sigs.shape[0]
        out = np.zeros((n_seg, 96), dtype=np.uint8)
        status = np.zeros(n_seg, dtype=np.int32)
        self._ck(self.lib.b2_aggregate(self.h, _p(sigs), _p(seg_off), n_seg, _p(out), _p(status)))
        return out, status

    def fast_aggregate_verify(self, members, off, bits, msgs32, sigs96):
        members, off, bits, n_agg, stride = self._batch(members, off, bits)
        msgs = _c(msgs32, np.uint8).reshape(n_agg, 32)
        sigs = _c(sigs96, np.uint8).reshape(n_agg, 96)
        ok = np.zeros(n_agg, dtype=np.uint8)
        self._ck(self.lib.b2_fast_aggregate_verify(self.h, _p(members), _p(off), _p(bits), stride, _p(msgs), _p(sigs), n_agg, _p(ok)))
        return ok

    def fast_aggregate_verify_pks(self, pks48, pk_off, msgs32, sigs96):
        pk_off = _c(pk_off, np.uint32)
        n_agg = pk_off.shape[0] - 1
        pks = _c(pks48, np.uint8).reshape(-1, 48)
        assert int(pk_off[-1]) == pks.shape[0]
        msgs = _c(msgs32, np.uint8).reshape(n_agg, 32)
        sigs = _c(sigs96, np.uint8).reshape(n_agg, 96)
        ok = np.zeros(n_agg, dtype=np.uint8)
        self._ck(self.lib.b2_fast_aggregate_verify_pks(self.h, _p(pks), _p(pk_off), _p(msgs), _p(sigs), n_agg, _p(ok)))
        return ok

    def aggregate_verify_pks(self, pks48, pair_off, msgs32, sigs96):
        """bls.AggregateVerify per set: set s = (pks48[i], msgs32[i]) for i in [pair_off[s], pair_off[s+1]), signature sigs96[s] -> uint8[n_sets]"""
        pair_off = _c(pair_off, np.uint32)
        n_sets = pair_off.shape[0] - 1
        pks = _c(pks48, np.uint8).reshape(-1, 48)
        msgs = _c(msgs32, np.uint8).reshape(-1, 32)
        assert int(pair_off[-1]) == pks.shape[0] == msgs.shape[0]
        sigs = _c(sigs96, np.uint8).reshape(n_sets, 96)
        ok = np.zeros(n_sets, dtype=np.uint8)
        self._ck(self.lib.b2_aggregate_verify_pks(self.h, _p(pks), _p(msgs), _p(pair_off), _p(sigs), n_sets, _p(ok)))
        return ok

    def aggregate_verify(self, signers, pair_off, msgs32, sigs96):
        """bls.AggregateVerify with the keys taken from the registry: pair i is (registry key signers[i], msgs32[i])"""
        pair_off = _c(pair_off, np.uint32)
        n_sets = pair_off.shape[0] - 1
        signers = _c(signers, np.uint32)
        msgs = _c(msgs32, np.uint8).reshape(-1, 32)
        assert int(pair_off[-1]) == signers.shape[0] == msgs.shape[0]
        sigs = _c(sigs96, np.uint8).reshape(n_sets, 96)
        ok = np.zeros(n_sets, dtype=np.uint8)
        self._ck(self.lib.b2_aggregate_verify(self.h, _p(signers), _p(msgs), _p(pair_off), _p(sigs), n_sets, _p(ok)))
        return ok

    def aggregate_pks(self, pks48, off):
        """bls.AggregatePKs per segment s = pks48[off[s] .. off[s+1]) -> (uint8[n_seg,48] compressed sums, uint8[n_seg] B2_PK_* status bits)"""
        off = _c(off, np.uint32)
        n_seg = off.shape[0] - 1
        pks = _c(pks48, np.uint8).reshape(-1, 48)
        assert int(off[-1]) == pks.shape[0]
        out = np.zeros((n_seg, 48), dtype=np.uint8)
        status = np.zeros(n_seg, dtype=np.uint8)
        self._ck(self.lib.b2_aggregate_pks(self.h, _p(pks), _p(off), n_seg, _p(out), _p(status)))
        return out, status

    # ------------------------------------------------------------------ sync committees (Altair process_sync_aggregate)
    def sync_committee_load(self, pubkeys48, committee_size: int):
        """n committees of committee_size keys, uint8[n * committee_size, 48] committee after committee: decoded, KeyValidated and
        summed once on the device (they replace the previously loaded committees).  Returns uint8[n * committee_size]: 1 where
        KeyValidate passed."""
        pk = _c(pubkeys48, np.uint8).reshape(-1, 48)
        size = int(committee_size)
        assert size > 0 and pk.shape[0] % size == 0
        valid = np.zeros(pk.shape[0], dtype=np.uint8)
        self._ck(self.lib.b2_sync_committee_load(self.h, _p(pk), size, pk.shape[0] // size, _p(valid)))
        self.sync_committee_size = size
        return valid

    def sync_aggregate_verify(self, committee_idx, bits, msgs32, sigs96, want_pubkeys: bool = False):
        """eth_fast_aggregate_verify per block: block i = participants of committee committee_idx[i] selected by its Bitvector row
        bits[i] (uint8[n, ceil(committee_size / 8)]), signing root msgs32[i], signature sigs96[i] -> uint8[n] verdicts, and with
        want_pubkeys also uint8[n, 48]: the compressed aggregate key of the participants."""
        cidx = _c(committee_idx, np.uint32)
        n = cidx.shape[0]
        b = _c(bits, np.uint8).reshape(n, -1)
        msgs = _c(msgs32, np.uint8).reshape(n, 32)
        sigs = _c(sigs96, np.uint8).reshape(n, 96)
        ok = np.zeros(n, dtype=np.uint8)
        pk = np.zeros((n, 48), dtype=np.uint8) if want_pubkeys else None
        self._ck(self.lib.b2_sync_aggregate_verify(self.h, _p(cidx), _p(b), _p(msgs), _p(sigs), n, _p(ok), _p(pk)))
        return (ok, pk) if want_pubkeys else ok

    @staticmethod
    def _sk_limbs(sks):
        out = np.zeros((len(sks), 8), dtype=np.uint32)
        for i, k in enumerate(sks):
            k = int(k)
            for j in range(8):
                out[i, j] = (k >> (32 * j)) & 0xFFFFFFFF
        return out

    def sk_to_pk(self, sks):
        sk8 = sks if isinstance(sks, np.ndarray) else self._sk_limbs(sks)
        sk8 = _c(sk8, np.uint32).reshape(-1, 8)
        out = np.zeros((sk8.shape[0], 48), dtype=np.uint8)
        self._ck(self.lib.b2_sk_to_pk(self.h, _p(sk8), sk8.shape[0], _p(out)))
        return out

    def sign(self, sks, msg_idx, msgs32):
        sk8 = sks if isinstance(sks, np.ndarray) else self._sk_limbs(sks)
        sk8 = _c(sk8, np.uint32).reshape(-1, 8)
        msg_idx = _c(msg_idx, np.uint32)
        msgs = _c(msgs32, np.uint8).reshape(-1, 32)
        out = np.zeros((sk8.shape[0], 96), dtype=np.uint8)
        self._ck(self.lib.b2_sign(self.h, _p(sk8), _p(msg_idx), sk8.shape[0], _p(msgs), msgs.shape[0], _p(out)))
        return out

    def hash_to_g2(self, msgs32):
        msgs = _c(msgs32, np.uint8).reshape(-1, 32)
        out = np.zeros((msgs.shape[0], 96), dtype=np.uint8)
        self._ck(self.lib.b2_hash_to_g2(self.h, _p(msgs), msgs.shape[0], _p(out)))
        return out

    def sha256_batch(self, msgs, msg_len: int):
        """SHA-256 of n fixed-length messages (uint8[n, msg_len]) on the GPU -> uint8[n, 32]."""
        m = _c(msgs, np.uint8).reshape(-1, msg_len) if msg_len else np.zeros((int(msgs), 0), dtype=np.uint8)
        n = m.shape[0]
        out = np.zeros((n, 32), dtype=np.uint8)
        self._ck(self.lib.b2_sha256_batch(self.h, _p(m) if msg_len else None, msg_len, n, _p(out)))
        return out

    # ------------------------------------------------------------------ hash_tree_root (pos-evolution.md:423, :1078)
    def ssz_validators_load(self, records) -> bytes:
        """Build the device tree of List[Validator, 2^40] from uint8[n, 121] SSZ-serialised records (spec.serialize_validators);
        returns its 32-byte root."""
        rec = _c(records, np.uint8).reshape(-1, 121)
        out = np.zeros(32, dtype=np.uint8)
        self._ck(self.lib.b2_ssz_validators_load(self.h, _p(rec), rec.shape[0], _p(out)))
        self.ssz_loads += 1
        return out.tobytes()

    def ssz_validators_update(self, idx, records) -> bytes:
        """Replace the records at idx (uint32, strictly increasing, below n) in the device tree and return the new root; re-hashes
        only those leaves and their paths."""
        idx = _c(idx, np.uint32)
        rec = _c(records, np.uint8).reshape(-1, 121)
        assert rec.shape[0] == idx.shape[0]
        out = np.zeros(32, dtype=np.uint8)
        self._ck(self.lib.b2_ssz_validators_update(self.h, _p(idx), _p(rec), idx.shape[0], _p(out)))
        return out.tobytes()

    def ssz_chunks_root(self, array, limit_depth: int, length=None) -> bytes:
        """Root of the bytes of `array` (little-endian basic values or 32-byte roots) packed into chunks and merkleized to depth
        limit_depth; with `length`, mix_in_length(root, length) -- the root of a List, without it of a Vector."""
        data = np.ascontiguousarray(array).view(np.uint8).reshape(-1)
        out = np.zeros(32, dtype=np.uint8)
        self._ck(self.lib.b2_ssz_chunks_root(self.h, _p(data), data.shape[0], limit_depth, int(length is not None),
                                             0 if length is None else int(length), _p(out)))
        return out.tobytes()

    def attestations_decode(self, wire: bytes, woff, bits_stride: int, max_bits: int):
        """SSZ wire decode of n Attestations (pos-evolution.md:714-717) -> (bits u8[n][stride], bit_len u32[n], data128 u8[n][128],
        sig96 u8[n][96], status i32[n])."""
        woff = _c(woff, np.uint32)
        n = woff.shape[0] - 1
        w = np.frombuffer(bytes(wire), dtype=np.uint8) if len(wire) else np.zeros(1, dtype=np.uint8)
        assert int(woff[-1]) == len(wire)
        bits = np.zeros((n, bits_stride), dtype=np.uint8)
        blen = np.zeros(n, dtype=np.uint32)
        data = np.zeros((n, 128), dtype=np.uint8)
        sig = np.zeros((n, 96), dtype=np.uint8)
        st = np.zeros(n, dtype=np.int32)
        self._ck(self.lib.b2_attestations_decode(self.h, _p(w), _p(woff), n, int(bits_stride), int(max_bits), _p(bits), _p(blen), _p(data), _p(sig), _p(st)))
        return bits, blen, data, sig, st

    def attestation_intake(self, wire: bytes, woff, off, epoch: int, current_slot: int, domain32: bytes, committees_per_slot: int,
                           slots_per_epoch: int, bits_stride: int, max_votes: int) -> IntakeResult:
        """One epoch of unaggregated Attestations (the wire form of attestations_decode) checked against the device tree and turned into
        the vote form's inputs (include/b200pos.h, b2_attestation_intake: statuses 0-13); committee c = members off[c] .. off[c+1]."""
        woff, off = _c(woff, np.uint32), _c(off, np.uint32)
        n_att, n_c = woff.shape[0] - 1, off.shape[0] - 1
        w = np.frombuffer(bytes(wire), dtype=np.uint8) if len(wire) else np.zeros(1, dtype=np.uint8)
        dom = np.frombuffer(bytes(domain32), dtype=np.uint8)
        assert dom.shape == (32,)
        n_sig, mv = int(off[-1]), int(max_votes)
        r = IntakeResult(np.zeros(n_att, np.int32), np.zeros(n_sig, np.uint32), np.zeros(n_c + 1, np.uint32), np.zeros((n_sig, 96), np.uint8),
                         np.zeros((mv, 128), np.uint8), np.zeros((mv, 32), np.uint8), np.zeros(mv, np.uint64), np.zeros(mv, np.uint64),
                         np.zeros(mv, np.uint32))
        self._ck(self.lib.b2_attestation_intake(self.h, _p(w), len(wire), _p(woff), n_att, _p(off), n_c, int(committees_per_slot),
                                                int(slots_per_epoch), int(bits_stride), int(epoch), int(current_slot), _p(dom), mv,
                                                *[_p(x) for x in r]))
        return r

    def single_attestation_intake(self, wire: bytes, woff, subnet, members, off, epoch: int, current_slot: int, domain32: bytes,
                                  committees_per_slot: int, slots_per_epoch: int, bits_stride: int, max_votes: int,
                                  subnet_count: int = 64) -> IntakeResult:
        """One epoch of Electra SingleAttestations (240-byte encodings back to back, woff their offsets, subnet the subnet each arrived
        on) checked against the device tree and turned into the vote form's inputs (include/b200pos.h, b2_single_attestation_intake:
        statuses 0-13); committee c = members[off[c] .. off[c+1]]; subnet_count = ATTESTATION_SUBNET_COUNT."""
        woff, subnet, members, off = _c(woff, np.uint32), _c(subnet, np.uint32), _c(members, np.uint32), _c(off, np.uint32)
        n_att, n_c = woff.shape[0] - 1, off.shape[0] - 1
        assert subnet.shape == (n_att,)
        w = np.frombuffer(bytes(wire), dtype=np.uint8) if len(wire) else np.zeros(1, dtype=np.uint8)
        mem = members if members.size else np.zeros(1, dtype=np.uint32)
        dom = np.frombuffer(bytes(domain32), dtype=np.uint8)
        assert dom.shape == (32,)
        n_sig, mv = int(off[-1]), int(max_votes)
        r = IntakeResult(np.zeros(n_att, np.int32), np.zeros(n_sig, np.uint32), np.zeros(n_c + 1, np.uint32), np.zeros((n_sig, 96), np.uint8),
                         np.zeros((mv, 128), np.uint8), np.zeros((mv, 32), np.uint8), np.zeros(mv, np.uint64), np.zeros(mv, np.uint64),
                         np.zeros(mv, np.uint32))
        self._ck(self.lib.b2_single_attestation_intake(self.h, _p(w), len(wire), _p(woff), n_att, _p(subnet), int(subnet_count), _p(mem), _p(off),
                                                       n_c, int(committees_per_slot), int(slots_per_epoch), int(bits_stride), int(epoch),
                                                       int(current_slot), _p(dom), mv, *[_p(x) for x in r]))
        return r

    def aggregate_and_proof_intake(self, wire: bytes, woff, members, off, epoch: int, current_slot: int, domains96: bytes,
                                   committees_per_slot: int, slots_per_epoch: int, bits_stride: int, target_aggregators: int = 16,
                                   propagation_slot_range: int = 32) -> AggregateIntakeResult:
        """One target epoch of SignedAggregateAndProof messages (SSZ encodings back to back, woff their offsets) checked and verified on
        the device (include/b200pos.h, b2_aggregate_and_proof_intake: statuses 0-20); committee c = members[off[c] .. off[c+1]].
        domains96 = the DOMAIN_BEACON_ATTESTER, DOMAIN_SELECTION_PROOF and DOMAIN_AGGREGATE_AND_PROOF domains of the epoch, back to back."""
        woff, members, off = _c(woff, np.uint32), _c(members, np.uint32), _c(off, np.uint32)
        n, n_c = woff.shape[0] - 1, off.shape[0] - 1
        w = np.frombuffer(bytes(wire), dtype=np.uint8) if len(wire) else np.zeros(1, dtype=np.uint8)
        mem = members if members.size else np.zeros(1, dtype=np.uint32)
        dom = np.frombuffer(bytes(domains96), dtype=np.uint8)
        assert dom.shape == (96,)
        width = 8 * int(bits_stride)
        r = AggregateIntakeResult(np.zeros(n, np.int32), np.zeros(n, np.uint32), np.zeros(n, np.uint32), np.zeros((n, bits_stride), np.uint8),
                                  np.zeros((n, 96), np.uint8), np.zeros((n, 32), np.uint8), np.zeros(n, np.uint64), np.zeros(n, np.uint32),
                                  np.zeros((n, width), np.uint32), np.zeros(n + 1, np.uint32))
        self._ck(self.lib.b2_aggregate_and_proof_intake(self.h, _p(w), len(wire), _p(woff), n, _p(mem), _p(off), n_c, int(committees_per_slot),
                                                        int(slots_per_epoch), int(bits_stride), int(epoch), int(current_slot), _p(dom),
                                                        int(target_aggregators), int(propagation_slot_range), *[_p(x) for x in r]))
        return r

    def block_attestations(self, wire: bytes, woff, block_off, block_slot, members, off, cps_prev: int, cps_cur: int, chain_roots,
                           justified80: bytes, domains64: bytes, slots_per_epoch: int, min_inclusion_delay: int, bits_stride: int,
                           increment: int, base_reward_per_increment: int) -> BlockAttestationsResult:
        """process_attestation for the attestations of a run of blocks of one epoch (include/b200pos.h, b2_block_attestations): the
        SSZ encodings back to back (woff their offsets), block b = attestations [block_off[b], block_off[b+1]) included at block_slot[b];
        committee c = members[off[c] .. off[c+1]], those of epoch e - 1 then those of e; chain_roots uint8[2 * slots_per_epoch, 32].
        Applies the blocks before the first invalid one to the device participation tables (both must be loaded)."""
        return self._block_attestations(self.lib.b2_block_attestations, (int(bits_stride),), wire, woff, block_off, block_slot, members, off,
                                        cps_prev, cps_cur, chain_roots, justified80, domains64, slots_per_epoch, min_inclusion_delay, increment,
                                        base_reward_per_increment)

    def block_attestations_electra(self, wire: bytes, woff, block_off, block_slot, members, off, cps_prev: int, cps_cur: int, chain_roots,
                                   justified80: bytes, domains64: bytes, slots_per_epoch: int, min_inclusion_delay: int,
                                   max_committees_per_slot: int, max_validators_per_committee: int, increment: int,
                                   base_reward_per_increment: int) -> BlockAttestationsResult:
        """block_attestations for Electra encodings (include/b200pos.h, b2_block_attestations_electra: statuses 0-13, Deneb's window and
        flags): an attestation names its committees of data.slot in committee_bits (max_committees_per_slot bits), and its Bitlist is their
        bit rows back to back.  Applies the blocks before the first invalid one to the device participation tables (both must be loaded)."""
        return self._block_attestations(self.lib.b2_block_attestations_electra, (int(max_committees_per_slot), int(max_validators_per_committee)),
                                        wire, woff, block_off, block_slot, members, off, cps_prev, cps_cur, chain_roots, justified80, domains64,
                                        slots_per_epoch, min_inclusion_delay, increment, base_reward_per_increment)

    def _block_attestations(self, fn, shape, wire, woff, block_off, block_slot, members, off, cps_prev, cps_cur, chain_roots, justified80,
                            domains64, slots_per_epoch, min_inclusion_delay, increment, base_reward_per_increment):
        """both host block-attestation calls: `shape` is what fn takes between min_inclusion_delay and the increment"""
        woff, block_off, members, off = _c(woff, np.uint32), _c(block_off, np.uint32), _c(members, np.uint32), _c(off, np.uint32)
        block_slot = _c(block_slot, np.uint64)
        roots = _c(chain_roots, np.uint8).reshape(-1)
        n, n_b = woff.shape[0] - 1, block_off.shape[0] - 1
        w = np.frombuffer(bytes(wire), dtype=np.uint8) if len(wire) else np.zeros(1, dtype=np.uint8)
        mem = members if members.size else np.zeros(1, dtype=np.uint32)
        j, dom = np.frombuffer(bytes(justified80), dtype=np.uint8), np.frombuffer(bytes(domains64), dtype=np.uint8)
        assert j.shape == (80,) and dom.shape == (64,) and roots.shape == (64 * int(slots_per_epoch),) and block_slot.shape == (max(n_b, 0),)
        r = BlockAttestationsResult(np.zeros(n, np.int32), np.zeros(n, np.uint8), np.zeros(n, np.uint64), np.zeros(n_b, np.int32),
                                    np.zeros(n_b, np.uint32), np.zeros(n_b, np.uint64), np.zeros(1, np.uint32))
        self._ck(fn(self.h, _p(w), len(wire), _p(woff), n, _p(block_off), _p(block_slot), n_b, _p(mem), _p(off), off.shape[0] - 1, int(cps_prev),
                    int(cps_cur), _p(roots), _p(j), _p(dom), int(slots_per_epoch), int(min_inclusion_delay), *shape, int(increment),
                    int(base_reward_per_increment), *[_p(x) for x in r]))
        return r._replace(n_applied=int(r.n_applied[0]))

    def sync_committee_messages(self, wire: bytes, woff, subnet, position_validator, subnet_count: int, current_slot: int,
                                domain32: bytes) -> SyncMessagesResult:
        """One slot of SyncCommitteeMessages (144-byte SSZ encodings back to back, woff their offsets; subnet[i] the topic's subnet id)
        checked and verified against the registry, grouped by root and aggregated (include/b200pos.h, b2_sync_committee_messages:
        statuses 0-6).  position_validator: the registry index of each sync committee position.  Per-root outputs are trimmed to n_roots."""
        woff, sub, pv = _c(woff, np.uint32), _c(subnet, np.uint32), _c(position_validator, np.uint32)
        n, size, count = woff.shape[0] - 1, pv.shape[0], int(subnet_count)
        assert sub.shape == (n,) and count > 0
        w = np.frombuffer(bytes(wire), dtype=np.uint8) if len(wire) else np.zeros(1, dtype=np.uint8)
        dom = np.frombuffer(bytes(domain32), dtype=np.uint8)
        assert dom.shape == (32,)
        sb, ab = (size // count + 7) // 8, (size + 7) // 8
        r = SyncMessagesResult(np.zeros(n, np.int32), np.zeros(n, np.uint32), np.zeros((n, 32), np.uint8), np.zeros((n, count, sb), np.uint8),
                               np.zeros((n, count, 96), np.uint8), np.zeros((n, count), np.uint8), np.zeros((n, ab), np.uint8),
                               np.zeros((n, 96), np.uint8))
        n_roots = np.zeros(1, np.uint32)
        self._ck(self.lib.b2_sync_committee_messages(self.h, _p(w), len(wire), _p(woff), n, _p(sub), _p(pv), size, count, int(current_slot),
                                                     _p(dom), _p(r.status), _p(r.root_id), _p(r.roots), _p(n_roots), _p(r.contrib_bits),
                                                     _p(r.contrib_sigs), _p(r.contrib_present), _p(r.agg_bits), _p(r.agg_sigs)))
        k = int(n_roots[0])
        return r._replace(roots=r.roots[:k], contrib_bits=r.contrib_bits[:k], contrib_sigs=r.contrib_sigs[:k], contrib_present=r.contrib_present[:k],
                          agg_bits=r.agg_bits[:k], agg_sigs=r.agg_sigs[:k])

    def sync_contribution_and_proof_intake(self, wire: bytes, woff, position_validator, subnet_count: int, current_slot: int, domains96: bytes,
                                           target_aggregators: int = 16) -> SyncContributionsResult:
        """One slot of SignedContributionAndProof messages (SSZ encodings back to back, woff their offsets) checked and verified against
        the registry, and each root's SyncAggregate built from its best contribution per subnet (include/b200pos.h,
        b2_sync_contribution_and_proof_intake: statuses 0-12).  position_validator: the registry index of each sync committee position;
        domains96: the DOMAIN_SYNC_COMMITTEE, DOMAIN_SYNC_COMMITTEE_SELECTION_PROOF and DOMAIN_CONTRIBUTION_AND_PROOF domains of current_slot's
        epoch, back to back.  Per-root outputs are trimmed to n_roots."""
        woff, pv = _c(woff, np.uint32), _c(position_validator, np.uint32)
        n, size, count = woff.shape[0] - 1, pv.shape[0], int(subnet_count)
        assert count > 0
        w = np.frombuffer(bytes(wire), dtype=np.uint8) if len(wire) else np.zeros(1, dtype=np.uint8)
        dom = np.frombuffer(bytes(domains96), dtype=np.uint8)
        assert dom.shape == (96,)
        ab = (size + 7) // 8
        r = SyncContributionsResult(np.zeros(n, np.int32), np.zeros(n, np.uint32), np.zeros((n, 32), np.uint8), np.zeros((n, count), np.uint32),
                                    np.zeros((n, ab), np.uint8), np.zeros((n, 96), np.uint8))
        n_roots = np.zeros(1, np.uint32)
        self._ck(self.lib.b2_sync_contribution_and_proof_intake(self.h, _p(w), len(wire), _p(woff), n, _p(pv), size, count, int(current_slot),
                                                                _p(dom), int(target_aggregators), _p(r.status), _p(r.root_id), _p(r.roots),
                                                                _p(n_roots), _p(r.best), _p(r.agg_bits), _p(r.agg_sigs)))
        k = int(n_roots[0])
        return r._replace(roots=r.roots[:k], best=r.best[:k], agg_bits=r.agg_bits[:k], agg_sigs=r.agg_sigs[:k])

    def signing_roots(self, data128, domains32):
        """compute_signing_root for n attestations: data128 uint8[n,128] (SSZ-serialised AttestationData), domains32 uint8[32] or uint8[n,32]."""
        d = _c(data128, np.uint8).reshape(-1, 128)
        dom = _c(domains32, np.uint8).reshape(-1, 32)
        n = d.shape[0]
        assert dom.shape[0] in (1, n)
        out = np.zeros((n, 32), dtype=np.uint8)
        self._ck(self.lib.b2_signing_roots(self.h, _p(d), _p(dom), 1 if dom.shape[0] == n and n > 1 else 0, n, _p(out)))
        return out

    def shuffle_committees(self, seed32: bytes, n_active: int, rounds: int, active=None):
        """members[i] = active[compute_shuffled_index(i, n_active, seed)] for the whole active set, on the GPU."""
        seed = np.frombuffer(bytes(seed32), dtype=np.uint8)
        assert seed.shape == (32,)
        act = _c(active, np.uint32) if active is not None else None
        out = np.zeros(n_active, dtype=np.uint32)
        self._ck(self.lib.b2_shuffle_committees(self.h, _p(seed), _p(act), n_active, rounds, _p(out)))
        return out

    # ------------------------------------------------------------------ fork choice
    def latest_messages_reset(self):
        self._ck(self.lib.b2_latest_messages_reset(self.h))

    def latest_messages_load(self, epoch, block_idx, has_msg, equivocating):
        e, b = _c(epoch, np.uint64), _c(block_idx, np.uint32)
        h, q = _c(has_msg, np.uint8), _c(equivocating, np.uint8)
        self._ck(self.lib.b2_latest_messages_load(self.h, _p(e), _p(b), _p(h), _p(q), e.shape[0]))

    def latest_messages_read(self):
        n = self.n_validators
        e, b, h = np.zeros(n, dtype=np.uint64), np.zeros(n, dtype=np.uint32), np.zeros(n, dtype=np.uint8)
        self._ck(self.lib.b2_latest_messages_read(self.h, _p(e), _p(b), _p(h), n))
        return e, b, h

    def latest_messages_update(self, members, off, bits, target_epoch, block_idx, accept=None):
        members, off, bits, n_agg, stride = self._batch(members, off, bits)
        te, bi = _c(target_epoch, np.uint64), _c(block_idx, np.uint32)
        acc = _c(accept, np.uint8) if accept is not None else None
        self._ck(self.lib.b2_latest_messages_update(self.h, _p(members), _p(off), _p(bits), stride, _p(te), _p(bi), _p(acc), n_agg))

    def participation_load(self, which: int, participation):
        p = _c(participation, np.uint8)
        self._ck(self.lib.b2_participation_load(self.h, int(which), _p(p), p.shape[0]))

    def participation_read(self, which: int):
        out = np.zeros(self.n_validators, dtype=np.uint8)
        self._ck(self.lib.b2_participation_read(self.h, int(which), _p(out), self.n_validators))
        return out

    def participation_update(self, which, members, off, bits, flag_mask, accept, increment, base_reward_per_increment):
        """process_attestation's flag loop (:745-749) for a batch; returns the per-attestation proposer_reward_numerator (u64)."""
        members, off, bits, n_agg, stride = self._batch(members, off, bits)
        fm = _c(flag_mask, np.uint8)
        acc = _c(accept, np.uint8) if accept is not None else None
        num = np.zeros(n_agg, dtype=np.uint64)
        self._ck(self.lib.b2_participation_update(self.h, int(which), _p(members), _p(off), _p(bits), stride, _p(fm), _p(acc), n_agg,
                                                  int(increment), int(base_reward_per_increment), _p(num)))
        return num

    def ffg_balances(self, flag_index: int):
        """(total_active, current_epoch_flag_balance, previous_epoch_flag_balance, total_active_unslashed) -- pos-evolution.md:793-803."""
        out = np.zeros(4, dtype=np.uint64)
        self._ck(self.lib.b2_ffg_balances(self.h, int(flag_index), _p(out)))
        return tuple(int(x) for x in out)

    def set_fork_choice_params(self, min_vote_epoch: int = 0, exclude_slashed: bool = False):
        self._ck(self.lib.b2_set_fork_choice_params(self.h, int(min_vote_epoch), 1 if exclude_slashed else 0))

    def set_verify_mode(self, rlc: bool, seed32: bytes = None):
        """FastAggregateVerify per aggregate (default) or in random-linear-combination batches of 32 with per-aggregate fallback
        (same verdict vector, about half the pairing work).  seed32: the verifier's secret randomness (os.urandom when None)."""
        import os
        seed = np.frombuffer(bytes(seed32) if seed32 is not None else os.urandom(32), dtype=np.uint8)
        assert seed.shape == (32,)
        self._ck(self.lib.b2_set_verify_mode(self.h, 1 if rlc else 0, _p(seed) if rlc else None))

    def on_attester_slashing(self, indices_1, indices_2):
        """Store.equivocating_indices |= set(indices_1) & set(indices_2)   (pos-evolution.md:1459-1461); both lists sorted."""
        a, b = _c(indices_1, np.uint32), _c(indices_2, np.uint32)
        self._ck(self.lib.b2_on_attester_slashing(self.h, _p(a), a.shape[0], _p(b), b.shape[0]))

    # ------------------------------------------------------------------ slasher (is_slashable_attestation_data, pos-evolution.md:1128-1143)
    def slasher_init(self, n_validators: int, history_epochs: int, max_attestations_per_target: int, current_epoch: int = 0,
                     v_begin: int = 0, v_end: int = None):
        """Device-resident attestation history of n_validators over a ring of history_epochs epochs (6 * n * H + 32 * H * max bytes);
        raises B2Error(B2_ENOMEM) without allocating when that exceeds the free device memory.  [v_begin, v_end): hold the validators
        of that range only (6 * (v_end - v_begin) * H + 32 * H * max bytes); members outside it are skipped silently."""
        v_end = n_validators if v_end is None else v_end
        self._ck(self.lib.b2_slasher_init_range(self.h, int(n_validators), int(v_begin), int(v_end), int(history_epochs),
                                                int(max_attestations_per_target), int(current_epoch)))

    def slasher_free(self):
        self._ck(self.lib.b2_slasher_free(self.h))

    def slasher_advance(self, current_epoch: int):
        self._ck(self.lib.b2_slasher_advance(self.h, int(current_epoch)))

    def slasher_update(self, members, off, bits, source_epoch, target_epoch, data_root32, accept=None):
        """Offer a batch of aggregates -> (status int32[n_agg] B2_SLASHER_*, kind uint8[len(members)] B2_SLASHABLE_* bits per member
        slot, conflict_target uint32[len(members), 2] (smallest surrounded / largest surrounding target, 0xffffffff = none), n_flagged)."""
        members, off, bits, n_agg, stride = self._batch(members, off, bits)
        se, te = _c(source_epoch, np.uint64), _c(target_epoch, np.uint64)
        roots = _c(data_root32, np.uint8).reshape(n_agg, 32)
        acc = _c(accept, np.uint8) if accept is not None else None
        assert se.shape == (n_agg,) and te.shape == (n_agg,) and members.shape[0] >= int(off[-1])
        total = int(off[-1])
        status = np.zeros(n_agg, dtype=np.int32)
        kind = np.zeros(total, dtype=np.uint8)
        conflict = np.full((total, 2), 0xFFFFFFFF, dtype=np.uint32)
        flagged = ctypes.c_uint32(0)
        self._ck(self.lib.b2_slasher_update(self.h, _p(members), _p(off), _p(bits), stride, _p(se), _p(te), _p(roots), _p(acc), n_agg,
                                            _p(status), _p(kind), _p(conflict), ctypes.byref(flagged)))
        return status, kind, conflict, int(flagged.value)

    # ------------------------------------------------------------------ equivocation discounting (pos-evolution.md:1405-1461)
    def slasher_discount(self, members, kind):
        """Every validator with a flagged member slot (kind != 0, the kind vector of slasher_update, members parallel to it) joins
        Store.equivocating_indices: its votes stop counting.  -> (new uint8[len(kind)]: 1 on exactly one slot of each validator this
        call newly marked, n_new)."""
        k = _c(kind, np.uint8)
        m = _c(members, np.uint32)[:k.shape[0]]
        assert m.shape == k.shape
        new = np.zeros(k.shape[0], dtype=np.uint8)
        n_new = ctypes.c_uint32(0)
        self._ck(self.lib.b2_slasher_discount(self.h, _p(m), _p(k), k.shape[0], _p(new), ctypes.byref(n_new)))
        return new, int(n_new.value)

    def equivocating(self):
        """Store.equivocating_indices as uint8[n_validators] (nonzero = equivocating)"""
        out = np.zeros(self.n_validators, dtype=np.uint8)
        self._ck(self.lib.b2_equivocating_read(self.h, _p(out), self.n_validators))
        return out

    # ------------------------------------------------------------------ block packing (BeaconBlockBody.attestations, pos-evolution.md:639)
    def pack_attestations(self, members, committee_off, committee_table, cand_committee, cand_data, cand_flag_mask, bits, sigs96, max_out: int,
                          increment: int, base_reward_per_increment: int) -> "PackResult":
        """Fold disjoint aggregates of one vote and pick up to max_out folded aggregates greedily by proposer-reward numerator against
        the device participation tables (include/b200pos.h, b2_pack_attestations).  bits: uint8[n_cand, bits_stride].  Returns a
        PackResult trimmed to the n_out picks, in pick order."""
        members, off = _c(members, np.uint32), _c(committee_off, np.uint32)
        table = _c(committee_table, np.uint8)
        cc, cd, cm = _c(cand_committee, np.uint32), _c(cand_data, np.uint32), _c(cand_flag_mask, np.uint8)
        n_cand, n_comm = cc.shape[0], off.shape[0] - 1
        b = _c(bits, np.uint8)
        b = b if b.ndim == 2 else b.reshape(n_cand, -1)
        stride = b.shape[1]
        sigs = _c(sigs96, np.uint8).reshape(n_cand, 96)
        assert table.shape == (n_comm,) and cd.shape == (n_cand,) and cm.shape == (n_cand,) and max_out > 0
        n_out = ctypes.c_uint32(0)
        o_comm, o_data = np.zeros(max_out, dtype=np.uint32), np.zeros(max_out, dtype=np.uint32)
        o_bits, o_sig = np.zeros((max_out, stride), dtype=np.uint8), np.zeros((max_out, 96), dtype=np.uint8)
        o_num, o_soff = np.zeros(max_out, dtype=np.uint64), np.zeros(max_out + 1, dtype=np.uint32)
        o_src, status = np.zeros(max(n_cand, 1), dtype=np.uint32), np.zeros(max(n_cand, 1), dtype=np.uint8)
        self._ck(self.lib.b2_pack_attestations(self.h, _p(members), _p(off), _p(table), n_comm, _p(cc), _p(cd), _p(cm), _p(b), stride, _p(sigs), n_cand,
                                               int(max_out), int(increment), int(base_reward_per_increment), ctypes.byref(n_out), _p(o_comm),
                                               _p(o_data), _p(o_bits), _p(o_sig), _p(o_num), _p(o_soff), _p(o_src), _p(status)))
        n = int(n_out.value)
        return PackResult(o_comm[:n], o_data[:n], o_bits[:n], o_num[:n], o_soff[:n + 1], o_src[:int(o_soff[n])], o_sig[:n], status[:n_cand])

    def pack_attestations_dev(self, d_members, d_committee_off, d_committee_table, d_cand_committee, d_cand_data, d_cand_flag_mask, d_bits, d_sigs,
                              max_out: int, increment: int, base_reward_per_increment: int, d_n_out, d_out_committee, d_out_data, d_out_bits,
                              d_out_sig, d_out_numerator, d_out_src_off, d_out_src, d_cand_status):
        """b2_pack_attestations_dev on torch CUDA tensors (asynchronous on the current stream; d_n_out uint32[1] is written on the device).
        Outputs sized as the host form before trimming: max_out rows, max_out + 1 offsets, n_cand sources and statuses."""
        n_cand = d_cand_committee.numel()
        self._ck(self.lib.b2_pack_attestations_dev(self.h, d_members.data_ptr(), d_committee_off.data_ptr(), d_committee_table.data_ptr(),
                                                   d_committee_off.numel() - 1, d_cand_committee.data_ptr(), d_cand_data.data_ptr(),
                                                   d_cand_flag_mask.data_ptr(), d_bits.data_ptr(), d_bits.shape[1], d_sigs.data_ptr(), n_cand,
                                                   int(max_out), int(increment), int(base_reward_per_increment), d_n_out.data_ptr(),
                                                   d_out_committee.data_ptr(), d_out_data.data_ptr(), d_out_bits.data_ptr(), d_out_sig.data_ptr(),
                                                   d_out_numerator.data_ptr(), d_out_src_off.data_ptr(), d_out_src.data_ptr(), d_cand_status.data_ptr(),
                                                   self._stream()))

    def tree_load(self, parent, slot, roots32, leaf_viable):
        parent, slot = _c(parent, np.uint32), _c(slot, np.uint64)
        roots = _c(roots32, np.uint8).reshape(-1, 32)
        viable = _c(leaf_viable, np.uint8)
        n = parent.shape[0]
        assert slot.shape == (n,) and roots.shape[0] == n and viable.shape == (n,)
        self._ck(self.lib.b2_tree_load(self.h, _p(parent), _p(slot), _p(roots), _p(viable), n))
        self.n_blocks = n

    def tree_add(self, parent, slot, roots32, leaf_viable):
        """Append k blocks to the loaded tree (ids n .. n+k-1, parent[j] < n + j); the arrays are those of tree_load."""
        parent, slot = _c(parent, np.uint32), _c(slot, np.uint64)
        roots = _c(roots32, np.uint8).reshape(-1, 32)
        viable = _c(leaf_viable, np.uint8)
        k = parent.shape[0]
        assert slot.shape == (k,) and roots.shape[0] == k and viable.shape == (k,)
        self._ck(self.lib.b2_tree_add(self.h, _p(parent), _p(slot), _p(roots), _p(viable), k))
        self.n_blocks += k

    def tree_prune(self, new_root: int):
        """Keep the subtree of block new_root, which becomes id 0; the latest messages are re-mapped on the device.  Returns the
        uint32 map old id -> new id (0xFFFFFFFF for a dropped block)."""
        m = np.zeros(self.n_blocks, dtype=np.uint32)
        self._ck(self.lib.b2_tree_prune(self.h, int(new_root), _p(m)))
        self.n_blocks = self.tree_size()
        return m

    def tree_set_viable(self, idx, viable):
        """Set the leaf-viability byte of blocks idx (the get_filtered_block_tree test)."""
        idx, viable = _c(idx, np.uint32), _c(viable, np.uint8)
        assert idx.shape == viable.shape and idx.ndim == 1
        self._ck(self.lib.b2_tree_set_viable(self.h, _p(idx), _p(viable), idx.shape[0]))

    def tree_size(self) -> int:
        return int(self.lib.b2_tree_size(self.h))

    def get_weights(self, boost_idx: int = -1, boost_score: int = 0):
        w = np.zeros(self.n_blocks, dtype=np.uint64)
        self._ck(self.lib.b2_get_weights(self.h, int(boost_idx), int(boost_score), _p(w)))
        return w

    def get_head(self, justified_idx: int = 0, boost_idx: int = -1, boost_score: int = 0) -> int:
        out = ctypes.c_uint32(0)
        self._ck(self.lib.b2_get_head(self.h, int(justified_idx), int(boost_idx), int(boost_score), ctypes.byref(out)))
        return int(out.value)

    # ------------------------------------------------------------------ multi-GPU get_head over NVLink peer memory
    def fc_exchange_setup(self, rank: int, world: int, process_group=None):
        """Map the vote-exchange blocks of all ranks of the box into this context (CUDA IPC handles all-gathered over `process_group`;
        world == 1 needs no group).  Call after tree_load, on every rank."""
        h = np.zeros(64, dtype=np.uint8)
        self._ck(self.lib.b2_fc_exchange_export(self.h, _p(h)))
        if world > 1:
            import torch.distributed as dist
            gathered = [None] * world
            dist.all_gather_object(gathered, h.tobytes(), group=process_group)
            allh = np.frombuffer(b"".join(gathered), dtype=np.uint8).copy()
        else:
            allh = h
        self._ck(self.lib.b2_fc_exchange_open(self.h, int(rank), int(world), _p(allh)))

    def get_head_multi(self, v_begin: int, v_end: int, justified_idx: int = 0, boost_idx: int = -1, boost_score: int = 0) -> int:
        """COLLECTIVE get_head: this rank scatters validators [v_begin, v_end); the all-reduce runs inside the kernel over NVLink."""
        out = ctypes.c_uint32(0)
        self._ck(self.lib.b2_get_head_multi(self.h, int(v_begin), int(v_end), int(justified_idx), int(boost_idx), int(boost_score), ctypes.byref(out)))
        return int(out.value)

    def debug_head_clocks(self):
        """clock64 stamps of the phases of the last get_head (profiling aid) -> uint64[32]; reading clears them (unwritten slots read 0)"""
        out = np.zeros(32, dtype=np.uint64)
        self._ck(self.lib.b2_debug_head_clocks(self.h, _p(out)))
        return out

    # ------------------------------------------------------------------ device-pointer entry points (torch CUDA tensors)
    @staticmethod
    def _stream():
        import torch
        return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)

    def aggregate_dev(self, d_sigs, d_seg_off, d_out96, d_status):
        n_seg = d_seg_off.numel() - 1
        n_sig = d_sigs.numel() // 96
        self._ck(self.lib.b2_aggregate_dev(self.h, d_sigs.data_ptr(), d_seg_off.data_ptr(), n_seg, n_sig, d_out96.data_ptr(),
                                           d_status.data_ptr(), self._stream()))

    def fast_aggregate_verify_dev(self, d_members, d_off, d_bits, d_msgs, d_sigs, d_ok):
        n_agg = d_off.numel() - 1
        stride = d_bits.shape[1]
        self._ck(self.lib.b2_fast_aggregate_verify_dev(self.h, d_members.data_ptr(), d_off.data_ptr(), d_bits.data_ptr(), stride,
                                                       d_msgs.data_ptr(), d_sigs.data_ptr(), n_agg, d_ok.data_ptr(), self._stream()))

    def aggregate_verify_dev(self, d_signer, d_msgs, d_pair_off, d_sigs, d_ok):
        """b2_aggregate_verify_dev: d_signer uint32[n_pairs], d_msgs uint8[n_pairs,32], d_pair_off uint32[n_sets+1], d_sigs uint8[n_sets,96]"""
        n_sets = d_pair_off.numel() - 1
        self._ck(self.lib.b2_aggregate_verify_dev(self.h, d_signer.data_ptr(), d_msgs.data_ptr(), d_pair_off.data_ptr(), d_signer.numel(),
                                                  d_sigs.data_ptr(), n_sets, d_ok.data_ptr(), self._stream()))

    def sync_aggregate_verify_dev(self, d_committee_idx, d_bits, d_msgs, d_sigs, d_ok, d_pk48=None):
        """b2_sync_aggregate_verify_dev: d_committee_idx uint32[n], d_bits uint8[n, ceil(committee_size / 8)], d_msgs uint8[n,32],
        d_sigs uint8[n,96], d_ok uint8[n], d_pk48 uint8[n,48] or None"""
        n = d_committee_idx.numel()
        self._ck(self.lib.b2_sync_aggregate_verify_dev(self.h, d_committee_idx.data_ptr(), d_bits.data_ptr(), d_msgs.data_ptr(), d_sigs.data_ptr(), n,
                                                       d_ok.data_ptr(), d_pk48.data_ptr() if d_pk48 is not None else None, self._stream()))

    def latest_messages_update_dev(self, d_members, d_off, d_bits, d_target_epoch, d_block_idx, d_accept):
        n_agg = d_off.numel() - 1
        self._ck(self.lib.b2_latest_messages_update_dev(self.h, d_members.data_ptr(), d_off.data_ptr(), d_bits.data_ptr(), d_bits.shape[1],
                                                        d_target_epoch.data_ptr(), d_block_idx.data_ptr(),
                                                        d_accept.data_ptr() if d_accept is not None else None, n_agg, self._stream()))

    def slasher_advance_dev(self, current_epoch: int):
        """b2_slasher_advance_dev on the current stream: the column reset is enqueued, nothing synchronises; updates enqueued later
        on this stream see the new window"""
        self._ck(self.lib.b2_slasher_advance_dev(self.h, int(current_epoch), self._stream()))

    def slasher_update_dev(self, d_members, d_off, d_bits, d_source_epoch, d_target_epoch, d_roots, d_accept, d_status, d_kind, d_conflict,
                           d_n_flagged):
        """b2_slasher_update_dev: the arrays of latest_messages_update_dev plus uint64 source epochs and uint8[n_agg, 32] data roots;
        outputs int32[n_agg], uint8[len(members)], uint32[len(members), 2] or None, uint32[1]"""
        n_agg = d_off.numel() - 1
        self._ck(self.lib.b2_slasher_update_dev(self.h, d_members.data_ptr(), d_off.data_ptr(), d_bits.data_ptr(), d_bits.shape[1],
                                                d_source_epoch.data_ptr(), d_target_epoch.data_ptr(), d_roots.data_ptr(),
                                                d_accept.data_ptr() if d_accept is not None else None, n_agg, d_status.data_ptr(),
                                                d_kind.data_ptr(), d_conflict.data_ptr() if d_conflict is not None else None,
                                                d_n_flagged.data_ptr(), self._stream()))

    def slasher_discount_dev(self, d_members, d_kind, d_new, d_n_new):
        """b2_slasher_discount_dev on the current stream: d_members uint32 and d_kind uint8 (slasher_update_dev's) per member slot ->
        d_new uint8 per slot, d_n_new uint32[1]"""
        self._ck(self.lib.b2_slasher_discount_dev(self.h, d_members.data_ptr(), d_kind.data_ptr(), d_kind.numel(), d_new.data_ptr(),
                                                  d_n_new.data_ptr(), self._stream()))

    def equivocating_slice_dev(self, v_begin: int, v_end: int, d_out):
        """the equivocating table's bytes [v_begin, v_end) -> d_out (uint8 device tensor), on the current stream"""
        self._ck(self.lib.b2_equivocating_slice_dev(self.h, int(v_begin), int(v_end), d_out.data_ptr(), self._stream()))

    def equivocating_merge_dev(self, v_begin: int, v_end: int, d_table):
        """equivocating[v_begin:v_end] |= d_table[:v_end - v_begin], on the current stream"""
        self._ck(self.lib.b2_equivocating_merge_dev(self.h, int(v_begin), int(v_end), d_table.data_ptr(), self._stream()))

    def epoch_dev(self, d_sigs, d_members, d_off, d_bits, d_msgs, d_target_epoch, d_block_idx, d_agg_sig, d_agg_status, d_ok):
        n_agg = d_off.numel() - 1
        self._ck(self.lib.b2_epoch_dev(self.h, d_sigs.data_ptr(), d_members.data_ptr(), d_off.data_ptr(), d_bits.data_ptr(), d_bits.shape[1],
                                       d_msgs.data_ptr(), d_target_epoch.data_ptr() if d_target_epoch is not None else None,
                                       d_block_idx.data_ptr() if d_block_idx is not None else None, n_agg, d_sigs.numel() // 96,
                                       d_agg_sig.data_ptr(), d_agg_status.data_ptr(), d_ok.data_ptr(), self._stream()))

    def epoch_start_dev(self, slot, d_sigs, d_members, d_off, d_bits, d_msgs, d_agg_status):
        n_agg = d_off.numel() - 1
        self._ck(self.lib.b2_epoch_start_dev(self.h, int(slot), d_sigs.data_ptr(), d_members.data_ptr(), d_off.data_ptr(), d_bits.data_ptr(),
                                             d_bits.shape[1], d_msgs.data_ptr(), n_agg, d_sigs.numel() // 96, d_agg_status.data_ptr(), self._stream()))

    def epoch_tail_dev(self, slot, d_members, d_off, d_bits, d_target_epoch, d_block_idx, d_agg_sig, d_agg_status, d_ok):
        n_agg = d_off.numel() - 1
        """d_target_epoch / d_block_idx None: no LMD update in the tail (sharded epoch: the caller applies it after the verdict exchange)."""
        self._ck(self.lib.b2_epoch_tail_dev(self.h, int(slot), d_members.data_ptr(), d_off.data_ptr(), d_bits.data_ptr(), d_bits.shape[1],
                                            d_target_epoch.data_ptr() if d_target_epoch is not None else None,
                                            d_block_idx.data_ptr() if d_block_idx is not None else None, n_agg, d_agg_sig.data_ptr(),
                                            d_agg_status.data_ptr(), d_ok.data_ptr()))

    def votes_group_dev(self, d_vote, d_vote_off, d_members, d_off, d_sigs, c_begin, c_end, d_sigs_out, d_members_out, d_pos_out, d_seg_off,
                        d_bits_out, d_agg_bits_out, d_seg_off_loc=None):
        """b2_votes_group_dev on the current stream: group committee order by vote (include/b200pos.h).  d_vote uint32[n_sig], d_vote_off
        uint32[n_committees+1], d_members / d_off the committees; d_sigs / d_sigs_out uint8[*, 96] the signatures of committees [c_begin,
        c_end); outputs d_members_out / d_pos_out uint32[n_sig], d_seg_off uint32[n_votes+1], d_bits_out / d_agg_bits_out uint8[n_votes,
        bits_stride] (n_votes and bits_stride from d_seg_off and d_bits_out), d_seg_off_loc the range's offsets over its own signatures."""
        n_votes, stride = d_seg_off.numel() - 1, d_bits_out.shape[1]
        assert d_bits_out.shape[0] >= n_votes and d_agg_bits_out.shape[1] == stride
        self._ck(self.lib.b2_votes_group_dev(self.h, d_vote.data_ptr(), d_vote_off.data_ptr(), n_votes, d_members.data_ptr(), d_off.data_ptr(),
                                             d_off.numel() - 1, d_members.numel(), stride, d_sigs.data_ptr(), int(c_begin), int(c_end),
                                             d_sigs_out.data_ptr(), d_members_out.data_ptr(), d_pos_out.data_ptr(), d_seg_off.data_ptr(),
                                             d_seg_off_loc.data_ptr() if d_seg_off_loc is not None else None, d_bits_out.data_ptr(),
                                             d_agg_bits_out.data_ptr(), self._stream()))

    def attestation_intake_dev(self, d_wire, d_woff, d_off, epoch: int, current_slot: int, domain32: bytes, committees_per_slot: int,
                               slots_per_epoch: int, bits_stride: int, d_status, d_vote, d_vote_off, d_sigs, d_data128, d_msgs, d_source_epoch,
                               d_target_epoch, d_block_idx):
        """attestation_intake on device tensors (the wire's length is d_wire.numel(); max_votes = d_msgs.shape[0]), asynchronous on the
        current stream."""
        dom = np.frombuffer(bytes(domain32), dtype=np.uint8)
        assert dom.shape == (32,)
        self._ck(self.lib.b2_attestation_intake_dev(self.h, d_wire.data_ptr(), d_wire.numel(), d_woff.data_ptr(), d_woff.numel() - 1,
                                                    d_off.data_ptr(), d_off.numel() - 1, d_vote.numel(), int(committees_per_slot),
                                                    int(slots_per_epoch), int(bits_stride), int(epoch), int(current_slot), _p(dom),
                                                    d_msgs.shape[0], d_status.data_ptr(), d_vote.data_ptr(), d_vote_off.data_ptr(),
                                                    d_sigs.data_ptr(), d_data128.data_ptr(), d_msgs.data_ptr(), d_source_epoch.data_ptr(),
                                                    d_target_epoch.data_ptr(), d_block_idx.data_ptr(), self._stream()))

    def single_attestation_intake_dev(self, d_wire, d_woff, d_subnet, d_members, d_off, epoch: int, current_slot: int, domain32: bytes,
                                      committees_per_slot: int, slots_per_epoch: int, bits_stride: int, d_status, d_vote, d_vote_off, d_sigs,
                                      d_data128, d_msgs, d_source_epoch, d_target_epoch, d_block_idx, subnet_count: int = 64):
        """single_attestation_intake on device tensors (d_subnet int32/uint32[n_att]; the wire's length is d_wire.numel(); max_votes =
        d_msgs.shape[0]; the outputs as attestation_intake_dev's), asynchronous on the current stream."""
        dom = np.frombuffer(bytes(domain32), dtype=np.uint8)
        assert dom.shape == (32,)
        n_att = d_woff.numel() - 1
        assert d_subnet.numel() == n_att and d_members.numel() == d_vote.numel()
        self._ck(self.lib.b2_single_attestation_intake_dev(self.h, d_wire.data_ptr(), d_wire.numel(), d_woff.data_ptr(), n_att,
                                                           d_subnet.data_ptr(), int(subnet_count), d_members.data_ptr(), d_off.data_ptr(),
                                                           d_off.numel() - 1, d_vote.numel(), int(committees_per_slot), int(slots_per_epoch),
                                                           int(bits_stride), int(epoch), int(current_slot), _p(dom), d_msgs.shape[0],
                                                           d_status.data_ptr(), d_vote.data_ptr(), d_vote_off.data_ptr(), d_sigs.data_ptr(),
                                                           d_data128.data_ptr(), d_msgs.data_ptr(), d_source_epoch.data_ptr(),
                                                           d_target_epoch.data_ptr(), d_block_idx.data_ptr(), self._stream()))

    def aggregate_and_proof_intake_dev(self, d_wire, d_woff, d_members, d_off, epoch: int, current_slot: int, domains96: bytes,
                                       committees_per_slot: int, slots_per_epoch: int, d_status, d_committee, d_data_id, d_bits, d_sigs, d_msgs,
                                       d_target_epoch, d_block_idx, d_members_out, d_item_off, target_aggregators: int = 16,
                                       propagation_slot_range: int = 32):
        """aggregate_and_proof_intake on device tensors, asynchronous on the current stream: n = d_woff.numel() - 1 items, the wire's
        length is d_wire.numel(), bits_stride = d_bits.shape[1].  Outputs: d_status int32[n], d_committee / d_data_id / d_block_idx
        uint32[n], d_bits uint8[n, bits_stride], d_sigs uint8[n, 96], d_msgs uint8[n, 32], d_target_epoch uint64[n], d_members_out
        uint32[n, 8 * bits_stride], d_item_off uint32[n + 1].  on_attestation of the accepted aggregates is then
        latest_messages_update_dev(d_members_out, d_item_off, d_bits, d_target_epoch, d_block_idx, (d_status == 0).to(torch.uint8))."""
        dom = np.frombuffer(bytes(domains96), dtype=np.uint8)
        assert dom.shape == (96,)
        n, stride = d_woff.numel() - 1, d_bits.shape[1]
        assert d_members_out.numel() == n * 8 * stride and d_item_off.numel() == n + 1
        self._ck(self.lib.b2_aggregate_and_proof_intake_dev(self.h, d_wire.data_ptr(), d_wire.numel(), d_woff.data_ptr(), n, d_members.data_ptr(),
                                                            d_off.data_ptr(), d_off.numel() - 1, d_members.numel(), int(committees_per_slot),
                                                            int(slots_per_epoch), int(stride), int(epoch), int(current_slot), _p(dom),
                                                            int(target_aggregators), int(propagation_slot_range), d_status.data_ptr(),
                                                            d_committee.data_ptr(), d_data_id.data_ptr(), d_bits.data_ptr(), d_sigs.data_ptr(),
                                                            d_msgs.data_ptr(), d_target_epoch.data_ptr(), d_block_idx.data_ptr(),
                                                            d_members_out.data_ptr(), d_item_off.data_ptr(), self._stream()))

    def block_attestations_dev(self, d_wire, d_woff, d_block_off, d_block_slot, d_members, d_off, cps_prev: int, cps_cur: int, d_chain_roots,
                               justified80: bytes, domains64: bytes, slots_per_epoch: int, min_inclusion_delay: int, bits_stride: int,
                               increment: int, base_reward_per_increment: int, d_status, d_flag_mask, d_numerator, d_block_status, d_block_first,
                               d_block_reward, d_n_applied):
        """block_attestations on device tensors, asynchronous on the current stream: n_att = d_woff.numel() - 1, n_blocks =
        d_block_off.numel() - 1, the wire's length is d_wire.numel(), n_sig = d_members.numel().  Outputs: d_status int32[n_att],
        d_flag_mask uint8[n_att], d_numerator uint64[n_att], d_block_status int32[n_blocks], d_block_first uint32[n_blocks], d_block_reward
        uint64[n_blocks], d_n_applied uint32[1]."""
        self._block_attestations_dev(self.lib.b2_block_attestations_dev, (int(bits_stride),), d_wire, d_woff, d_block_off, d_block_slot, d_members,
                                     d_off, cps_prev, cps_cur, d_chain_roots, justified80, domains64, slots_per_epoch, min_inclusion_delay, increment,
                                     base_reward_per_increment, BlockAttestationsResult(d_status, d_flag_mask, d_numerator, d_block_status,
                                                                                        d_block_first, d_block_reward, d_n_applied))

    def block_attestations_electra_dev(self, d_wire, d_woff, d_block_off, d_block_slot, d_members, d_off, cps_prev: int, cps_cur: int,
                                       d_chain_roots, justified80: bytes, domains64: bytes, slots_per_epoch: int, min_inclusion_delay: int,
                                       max_committees_per_slot: int, max_validators_per_committee: int, row_max: int, increment: int,
                                       base_reward_per_increment: int, out=None) -> BlockAttestationsResult:
        """block_attestations_electra on device tensors, asynchronous on the current stream: n_att = d_woff.numel() - 1, n_blocks =
        d_block_off.numel() - 1, the wire's length is d_wire.numel(), n_sig = d_members.numel(); row_max, the largest member count of one
        slot's committees.  `out`: a BlockAttestationsResult of device tensors (status int32[n_att], flag_mask uint8[n_att], numerator
        uint64[n_att], block_status int32[n_blocks], block_first uint32[n_blocks], block_reward uint64[n_blocks], n_applied uint32[1]), or
        None to allocate them here.  Returns the outputs."""
        if out is None:
            import torch
            n, nb = d_woff.numel() - 1, d_block_off.numel() - 1
            z = lambda k, dt: torch.zeros(k, dtype=dt, device=d_woff.device)      # noqa: E731
            out = BlockAttestationsResult(z(n, torch.int32), z(n, torch.uint8), z(n, torch.uint64), z(nb, torch.int32), z(nb, torch.uint32),
                                          z(nb, torch.uint64), z(1, torch.uint32))
        shape = (int(max_committees_per_slot), int(max_validators_per_committee), int(row_max))
        self._block_attestations_dev(self.lib.b2_block_attestations_electra_dev, shape, d_wire, d_woff, d_block_off, d_block_slot, d_members, d_off,
                                     cps_prev, cps_cur, d_chain_roots, justified80, domains64, slots_per_epoch, min_inclusion_delay, increment,
                                     base_reward_per_increment, out)
        return out

    def _block_attestations_dev(self, fn, shape, d_wire, d_woff, d_block_off, d_block_slot, d_members, d_off, cps_prev, cps_cur, d_chain_roots,
                                justified80, domains64, slots_per_epoch, min_inclusion_delay, increment, base_reward_per_increment, out):
        """both device block-attestation calls: `shape` as in _block_attestations, `out` a BlockAttestationsResult of device tensors"""
        j, dom = np.frombuffer(bytes(justified80), dtype=np.uint8), np.frombuffer(bytes(domains64), dtype=np.uint8)
        assert j.shape == (80,) and dom.shape == (64,)
        self._ck(fn(self.h, d_wire.data_ptr(), d_wire.numel(), d_woff.data_ptr(), d_woff.numel() - 1, d_block_off.data_ptr(), d_block_slot.data_ptr(),
                    d_block_off.numel() - 1, d_members.data_ptr(), d_off.data_ptr(), d_off.numel() - 1, d_members.numel(), int(cps_prev), int(cps_cur),
                    d_chain_roots.data_ptr(), _p(j), _p(dom), int(slots_per_epoch), int(min_inclusion_delay), *shape, int(increment),
                    int(base_reward_per_increment), *[x.data_ptr() for x in out], self._stream()))

    def sync_committee_messages_dev(self, d_wire, d_woff, d_subnet, d_position_validator, subnet_count: int, current_slot: int, domain32: bytes,
                                    out=None, trim: bool = True) -> SyncMessagesResult:
        """sync_committee_messages on device tensors (n = d_woff.numel() - 1, the wire's length is d_wire.numel(), committee_size =
        d_position_validator.numel()), enqueued on the current stream.  `out`: (SyncMessagesResult of device tensors shaped as the host
        form's untrimmed outputs, n_roots tensor of 4 bytes), or None to allocate them here (status and root_id int32: a message that was
        not accepted has root id -1).  With trim (the default) the call waits for n_roots and returns the result with the per-root outputs
        trimmed to it; with trim=False it stays asynchronous and returns the pair `out` takes."""
        import torch
        dom = np.frombuffer(bytes(domain32), dtype=np.uint8)
        assert dom.shape == (32,)
        n, size, count = d_woff.numel() - 1, d_position_validator.numel(), int(subnet_count)
        assert d_subnet.numel() == n and count > 0
        sb, ab = (size // count + 7) // 8, (size + 7) // 8
        if out is None:
            dev, u8 = d_woff.device, torch.uint8
            out = SyncMessagesResult(torch.empty(n, dtype=torch.int32, device=dev), torch.empty(n, dtype=torch.int32, device=dev),
                                     torch.empty((n, 32), dtype=u8, device=dev), torch.empty((n, count, sb), dtype=u8, device=dev),
                                     torch.empty((n, count, 96), dtype=u8, device=dev), torch.empty((n, count), dtype=u8, device=dev),
                                     torch.empty((n, ab), dtype=u8, device=dev), torch.empty((n, 96), dtype=u8, device=dev))
            n_roots = torch.empty(1, dtype=torch.int32, device=dev)
        else:
            out, n_roots = out
        self._ck(self.lib.b2_sync_committee_messages_dev(self.h, d_wire.data_ptr(), d_wire.numel(), d_woff.data_ptr(), n, d_subnet.data_ptr(),
                                                         d_position_validator.data_ptr(), size, count, int(current_slot), _p(dom),
                                                         *[x.data_ptr() for x in out[:3]], n_roots.data_ptr(),
                                                         *[x.data_ptr() for x in out[3:]], self._stream()))
        if not trim:
            return out, n_roots
        k = int(n_roots.item())
        return out._replace(roots=out.roots[:k], contrib_bits=out.contrib_bits[:k], contrib_sigs=out.contrib_sigs[:k],
                            contrib_present=out.contrib_present[:k], agg_bits=out.agg_bits[:k], agg_sigs=out.agg_sigs[:k])

    def sync_contribution_and_proof_intake_dev(self, d_wire, d_woff, d_position_validator, subnet_count: int, current_slot: int,
                                               domains96: bytes, target_aggregators: int = 16, out=None,
                                               trim: bool = True) -> SyncContributionsResult:
        """sync_contribution_and_proof_intake on device tensors (n = d_woff.numel() - 1, the wire's length is d_wire.numel(), committee_size
        = d_position_validator.numel()), enqueued on the current stream.  `out`: (SyncContributionsResult of device tensors shaped as the
        host form's untrimmed outputs, n_roots tensor of 4 bytes), or None to allocate them here (status, root_id and best int32: none is -1).
        With trim (the default) the call waits for n_roots and returns the result with the per-root outputs trimmed to it; with trim=False
        it stays asynchronous and returns the pair `out` takes."""
        import torch
        dom = np.frombuffer(bytes(domains96), dtype=np.uint8)
        assert dom.shape == (96,)
        n, size, count = d_woff.numel() - 1, d_position_validator.numel(), int(subnet_count)
        assert count > 0
        if out is None:
            dev, u8, i32 = d_woff.device, torch.uint8, torch.int32
            out = SyncContributionsResult(torch.empty(n, dtype=i32, device=dev), torch.empty(n, dtype=i32, device=dev),
                                          torch.empty((n, 32), dtype=u8, device=dev), torch.empty((n, count), dtype=i32, device=dev),
                                          torch.empty((n, (size + 7) // 8), dtype=u8, device=dev), torch.empty((n, 96), dtype=u8, device=dev))
            n_roots = torch.empty(1, dtype=i32, device=dev)
        else:
            out, n_roots = out
        self._ck(self.lib.b2_sync_contribution_and_proof_intake_dev(self.h, d_wire.data_ptr(), d_wire.numel(), d_woff.data_ptr(), n,
                                                                    d_position_validator.data_ptr(), size, count, int(current_slot), _p(dom),
                                                                    int(target_aggregators), *[x.data_ptr() for x in out[:3]],
                                                                    n_roots.data_ptr(), *[x.data_ptr() for x in out[3:]], self._stream()))
        if not trim:
            return out, n_roots
        k = int(n_roots.item())
        return out._replace(roots=out.roots[:k], best=out.best[:k], agg_bits=out.agg_bits[:k], agg_sigs=out.agg_sigs[:k])

    def votes_empty_dev(self, d_bits, d_agg_sig, d_agg_status=None):
        """b2_votes_empty_dev on the current stream: every vote whose grouped bit row d_bits (uint8[n_votes, bits_stride]) has no attester
        gets 96 zero bytes in d_agg_sig and, when given, status 2 in d_agg_status"""
        self._ck(self.lib.b2_votes_empty_dev(self.h, d_bits.data_ptr(), d_bits.shape[1], d_bits.shape[0], d_agg_sig.data_ptr(),
                                             d_agg_status.data_ptr() if d_agg_status is not None else None, self._stream()))

    def epoch_set_pairing_form(self, team: bool):
        self._ck(self.lib.b2_epoch_set_pairing_form(self.h, 1 if team else 0))

    def epoch_wait_dev(self, slot):
        self._ck(self.lib.b2_epoch_wait_dev(self.h, int(slot), self._stream()))

    def vote_weights_dev(self, d_votes):
        self._ck(self.lib.b2_vote_weights_dev(self.h, d_votes.data_ptr(), self._stream()))

    def vote_weights_range_dev(self, v_begin, v_end, d_votes):
        """direct votes of the validators [v_begin, v_end) only (this rank's shard of one validator set)"""
        self._ck(self.lib.b2_vote_weights_range_dev(self.h, int(v_begin), int(v_end), d_votes.data_ptr(), self._stream()))

    def gather_probe_dev(self, d_members, d_off, d_bits, d_checksum, tma: bool = True):
        """gather stage of K2 alone: d_checksum[a] = XOR of the pubkey-record words aggregate a selects (TMA-staged or plain-load form)"""
        n_agg = d_off.numel() - 1
        self._ck(self.lib.b2_gather_probe_dev(self.h, d_members.data_ptr(), d_off.data_ptr(), d_bits.data_ptr(), d_bits.shape[1], n_agg,
                                              1 if tma else 0, d_checksum.data_ptr(), self._stream()))

    def guard_flags(self) -> int:
        """synchronise; return and clear the device-side input guard word (B2_GUARD_* bits) of the *_dev entry points"""
        out = ctypes.c_uint32(0)
        self._ck(self.lib.b2_guard_flags(self.h, ctypes.byref(out)))
        return int(out.value)

    def head_from_votes_dev(self, d_votes, d_head, justified_idx=0, boost_idx=-1, boost_score=0, d_weight=None):
        self._ck(self.lib.b2_head_from_votes_dev(self.h, d_votes.data_ptr(), int(justified_idx), int(boost_idx), int(boost_score),
                                                 d_weight.data_ptr() if d_weight is not None else None, d_head.data_ptr(), self._stream()))
