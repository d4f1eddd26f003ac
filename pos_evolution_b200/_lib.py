"""ctypes binding of libb200pos.so (include/b200pos.h).  There is no CPU fallback: if the shared
library is missing, or no sm_90 (H100) GPU is visible, importing callers get a loud error."""
import ctypes
import os
from ctypes import POINTER, c_char_p, c_int, c_int32, c_uint8, c_uint32, c_uint64, c_void_p

HERE = os.path.dirname(os.path.abspath(__file__))
# B2_LIB: load another build of the SAME library (tools/sanitize.sh: the ASan/UBSan-instrumented host side); not a fallback
LIB_PATH = os.environ.get("B2_LIB") or os.path.join(HERE, "libb200pos.so")

B2_OK, B2_EINVAL, B2_ECUDA, B2_ENODEVICE, B2_ENOMEM = 0, -1, -2, -3, -4
_ERRNAMES = {B2_EINVAL: "B2_EINVAL", B2_ECUDA: "B2_ECUDA", B2_ENODEVICE: "B2_ENODEVICE", B2_ENOMEM: "B2_ENOMEM"}


class B2Error(RuntimeError):
    def __init__(self, code, text):
        super().__init__("%s: %s" % (_ERRNAMES.get(code, code), text))
        self.code = code


_lib = None

u8p, u32p, u64p, i32p = POINTER(c_uint8), POINTER(c_uint32), POINTER(c_uint64), POINTER(c_int32)

# name -> (restype, argtypes); every symbol include/b200pos.h declares
SIGNATURES = {
    "b2_init": (c_int, [c_int, POINTER(c_void_p)]),
    "b2_destroy": (None, [c_void_p]),
    "b2_last_error": (c_char_p, [c_void_p]),
    "b2_sync": (c_int, [c_void_p]),
    "b2_launch_count": (c_uint64, [c_void_p]),
    "b2_registry_load": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_uint64, c_void_p]),
    "b2_key_validate": (c_int, [c_void_p, c_void_p, c_uint64, c_void_p]),
    "b2_registry_update_balances": (c_int, [c_void_p, c_void_p, c_void_p, c_uint64]),
    "b2_g1_aggregate": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_uint32, c_uint32, c_void_p, c_void_p]),
    "b2_aggregate": (c_int, [c_void_p, c_void_p, c_void_p, c_uint32, c_void_p, c_void_p]),
    "b2_fast_aggregate_verify": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_uint32, c_void_p, c_void_p, c_uint32, c_void_p]),
    "b2_fast_aggregate_verify_pks": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_uint32, c_void_p]),
    "b2_aggregate_verify_pks": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_uint32, c_void_p]),
    "b2_aggregate_verify": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_uint32, c_void_p]),
    "b2_aggregate_verify_dev": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_uint64, c_void_p, c_uint32, c_void_p, c_void_p]),
    "b2_aggregate_pks": (c_int, [c_void_p, c_void_p, c_void_p, c_uint32, c_void_p, c_void_p]),
    "b2_sync_committee_load": (c_int, [c_void_p, c_void_p, c_uint32, c_uint32, c_void_p]),
    "b2_sync_aggregate_verify": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_uint32, c_void_p, c_void_p]),
    "b2_sync_aggregate_verify_dev": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_uint32, c_void_p, c_void_p, c_void_p]),
    "b2_sk_to_pk": (c_int, [c_void_p, c_void_p, c_uint64, c_void_p]),
    "b2_sign": (c_int, [c_void_p, c_void_p, c_void_p, c_uint64, c_void_p, c_uint32, c_void_p]),
    "b2_hash_to_g2": (c_int, [c_void_p, c_void_p, c_uint32, c_void_p]),
    "b2_sha256_batch": (c_int, [c_void_p, c_void_p, c_uint32, c_uint64, c_void_p]),
    "b2_signing_roots": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_uint32, c_void_p]),
    "b2_shuffle_committees": (c_int, [c_void_p, c_void_p, c_void_p, c_uint32, c_uint32, c_void_p]),
    "b2_shuffle_committees_dev": (c_int, [c_void_p, c_void_p, c_void_p, c_uint32, c_uint32, c_void_p, c_void_p]),
    "b2_latest_messages_reset": (c_int, [c_void_p]),
    "b2_latest_messages_load": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_uint64]),
    "b2_latest_messages_read": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_uint64]),
    "b2_latest_messages_update": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_uint32, c_void_p, c_void_p, c_void_p, c_uint32]),
    "b2_participation_load": (c_int, [c_void_p, c_int, c_void_p, c_uint64]),
    "b2_participation_read": (c_int, [c_void_p, c_int, c_void_p, c_uint64]),
    "b2_participation_update": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_uint32, c_void_p, c_void_p, c_uint32, c_uint64, c_uint64, c_void_p]),
    "b2_ffg_balances": (c_int, [c_void_p, c_uint32, c_void_p]),
    "b2_attestations_decode": (c_int, [c_void_p, c_void_p, c_void_p, c_uint32, c_uint32, c_uint32, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "b2_set_fork_choice_params": (c_int, [c_void_p, c_uint64, c_int]),
    "b2_set_verify_mode": (c_int, [c_void_p, c_int, c_void_p]),
    "b2_epoch_set_pairing_form": (c_int, [c_void_p, c_int]),
    "b2_on_attester_slashing": (c_int, [c_void_p, c_void_p, c_uint32, c_void_p, c_uint32]),
    "b2_slasher_init": (c_int, [c_void_p, c_uint64, c_uint32, c_uint32, c_uint64]),
    "b2_slasher_free": (c_int, [c_void_p]),
    "b2_slasher_init_range": (c_int, [c_void_p, c_uint64, c_uint64, c_uint64, c_uint32, c_uint32, c_uint64]),
    "b2_slasher_advance": (c_int, [c_void_p, c_uint64]),
    "b2_slasher_advance_dev": (c_int, [c_void_p, c_uint64, c_void_p]),
    "b2_slasher_update": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_uint32, c_void_p, c_void_p, c_void_p, c_void_p, c_uint32,
                                  c_void_p, c_void_p, c_void_p, c_void_p]),
    "b2_slasher_update_dev": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_uint32, c_void_p, c_void_p, c_void_p, c_void_p, c_uint32,
                                      c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "b2_slasher_discount_dev": (c_int, [c_void_p, c_void_p, c_void_p, c_uint64, c_void_p, c_void_p, c_void_p]),
    "b2_slasher_discount": (c_int, [c_void_p, c_void_p, c_void_p, c_uint64, c_void_p, c_void_p]),
    "b2_equivocating_read": (c_int, [c_void_p, c_void_p, c_uint64]),
    "b2_equivocating_slice_dev": (c_int, [c_void_p, c_uint64, c_uint64, c_void_p, c_void_p]),
    "b2_equivocating_merge_dev": (c_int, [c_void_p, c_uint64, c_uint64, c_void_p, c_void_p]),
    "b2_pack_attestations":(c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_uint32, c_void_p, c_void_p, c_void_p, c_void_p, c_uint32, c_void_p,
                                     c_uint32, c_uint32, c_uint64, c_uint64, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                     c_void_p, c_void_p]),
    "b2_pack_attestations_dev": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_uint32, c_void_p, c_void_p, c_void_p, c_void_p, c_uint32,
                                         c_void_p, c_uint32, c_uint32, c_uint64, c_uint64, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                         c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "b2_tree_load": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_uint32]),
    "b2_tree_add": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_uint32]),
    "b2_tree_prune": (c_int, [c_void_p, c_uint32, c_void_p]),
    "b2_tree_set_viable": (c_int, [c_void_p, c_void_p, c_void_p, c_uint32]),
    "b2_get_weights": (c_int, [c_void_p, c_int32, c_uint64, c_void_p]),
    "b2_get_head": (c_int, [c_void_p, c_uint32, c_int32, c_uint64, c_void_p]),
    "b2_aggregate_dev": (c_int, [c_void_p, c_void_p, c_void_p, c_uint32, c_uint64, c_void_p, c_void_p, c_void_p]),
    "b2_fast_aggregate_verify_dev": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_uint32, c_void_p, c_void_p, c_uint32, c_void_p, c_void_p]),
    "b2_latest_messages_update_dev": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_uint32, c_void_p, c_void_p, c_void_p, c_uint32, c_void_p]),
    "b2_epoch_dev": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_uint32, c_void_p, c_void_p, c_void_p, c_uint32, c_uint64,
                             c_void_p, c_void_p, c_void_p, c_void_p]),
    "b2_epoch_start_dev": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_uint32, c_void_p, c_uint32, c_uint64, c_void_p, c_void_p]),
    "b2_epoch_tail_dev": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_uint32, c_void_p, c_void_p, c_uint32, c_void_p, c_void_p, c_void_p]),
    "b2_epoch_wait_dev": (c_int, [c_void_p, c_int, c_void_p]),
    "b2_votes_group_dev": (c_int, [c_void_p, c_void_p, c_void_p, c_uint32, c_void_p, c_void_p, c_uint32, c_uint64, c_uint32, c_void_p, c_uint32,
                                   c_uint32, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "b2_votes_empty_dev": (c_int, [c_void_p, c_void_p, c_uint32, c_uint32, c_void_p, c_void_p, c_void_p]),
    "b2_attestation_intake_dev": (c_int, [c_void_p, c_void_p, c_uint64, c_void_p, c_uint32, c_void_p, c_uint32, c_uint64, c_uint32, c_uint32,
                                          c_uint32, c_uint64, c_uint64, c_void_p, c_uint32, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                          c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "b2_attestation_intake": (c_int, [c_void_p, c_void_p, c_uint64, c_void_p, c_uint32, c_void_p, c_uint32, c_uint32, c_uint32, c_uint32, c_uint64,
                                      c_uint64, c_void_p, c_uint32, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                      c_void_p]),
    # ctx, wire, wire_len, woff, n_att, subnet, subnet_count, members, off, n_committees, [n_sig,] committees_per_slot, slots_per_epoch,
    # bits_stride, epoch, current_slot, domain32, max_votes, nine outputs[, stream]
    "b2_single_attestation_intake_dev": (c_int, [c_void_p, c_void_p, c_uint64, c_void_p, c_uint32, c_void_p, c_uint32, c_void_p, c_void_p, c_uint32,
                                                 c_uint64, c_uint32, c_uint32, c_uint32, c_uint64, c_uint64, c_void_p, c_uint32] + [c_void_p] * 10),
    "b2_single_attestation_intake": (c_int, [c_void_p, c_void_p, c_uint64, c_void_p, c_uint32, c_void_p, c_uint32, c_void_p, c_void_p, c_uint32,
                                             c_uint32, c_uint32, c_uint32, c_uint64, c_uint64, c_void_p, c_uint32] + [c_void_p] * 9),
    # ctx, wire, wire_len, woff, n, members, off, n_committees, [n_sig,] committees_per_slot, slots_per_epoch, bits_stride, epoch, current_slot,
    # domains96, target_aggregators, propagation_slot_range, ten outputs[, stream]
    "b2_aggregate_and_proof_intake_dev": (c_int, [c_void_p, c_void_p, c_uint64, c_void_p, c_uint32, c_void_p, c_void_p, c_uint32, c_uint64, c_uint32,
                                                  c_uint32, c_uint32, c_uint64, c_uint64, c_void_p, c_uint32, c_uint64] + [c_void_p] * 11),
    "b2_aggregate_and_proof_intake": (c_int, [c_void_p, c_void_p, c_uint64, c_void_p, c_uint32, c_void_p, c_void_p, c_uint32, c_uint32, c_uint32,
                                              c_uint32, c_uint64, c_uint64, c_void_p, c_uint32, c_uint64] + [c_void_p] * 10),
    # ctx, wire, wire_len, woff, n_att, block_off, block_slot, n_blocks, members, off, n_committees, [n_sig,] cps_prev, cps_cur, chain_roots, justified80,
    # domains64, slots_per_epoch, min_inclusion_delay, bits_stride, increment, base_reward_per_increment, seven outputs[, stream]
    "b2_block_attestations_dev": (c_int, [c_void_p, c_void_p, c_uint64, c_void_p, c_uint32, c_void_p, c_void_p, c_uint32, c_void_p, c_void_p, c_uint32,
                                          c_uint64, c_uint32, c_uint32, c_void_p, c_void_p, c_void_p, c_uint32, c_uint32, c_uint32, c_uint64,
                                          c_uint64] + [c_void_p] * 8),
    "b2_block_attestations": (c_int, [c_void_p, c_void_p, c_uint64, c_void_p, c_uint32, c_void_p, c_void_p, c_uint32, c_void_p, c_void_p,
                                      c_uint32, c_uint32, c_uint32, c_void_p, c_void_p, c_void_p, c_uint32, c_uint32, c_uint32, c_uint64, c_uint64] + [c_void_p] * 7),
    # ctx, wire, wire_len, woff, n_att, block_off, block_slot, n_blocks, members, off, n_committees, [n_sig,] cps_prev, cps_cur, chain_roots, justified80,
    # domains64, slots_per_epoch, min_inclusion_delay, max_committees_per_slot, max_validators_per_committee, [row_max,] increment,
    # base_reward_per_increment, seven outputs[, stream]
    "b2_block_attestations_electra_dev": (c_int, [c_void_p, c_void_p, c_uint64, c_void_p, c_uint32, c_void_p, c_void_p, c_uint32, c_void_p, c_void_p,
                                                  c_uint32, c_uint64, c_uint32, c_uint32, c_void_p, c_void_p, c_void_p, c_uint32, c_uint32, c_uint32,
                                                  c_uint32, c_uint32, c_uint64, c_uint64] + [c_void_p] * 8),
    "b2_block_attestations_electra": (c_int, [c_void_p, c_void_p, c_uint64, c_void_p, c_uint32, c_void_p, c_void_p, c_uint32, c_void_p, c_void_p,
                                              c_uint32, c_uint32, c_uint32, c_void_p, c_void_p, c_void_p, c_uint32, c_uint32, c_uint32, c_uint32,
                                              c_uint64, c_uint64] + [c_void_p] * 7),
    # ctx, wire, wire_len, woff, n, subnet, position_validator, committee_size, subnet_count, current_slot, domain32, nine outputs[, stream]
    "b2_sync_committee_messages_dev": (c_int, [c_void_p, c_void_p, c_uint64, c_void_p, c_uint32, c_void_p, c_void_p, c_uint32, c_uint32, c_uint64,
                                               c_void_p] + [c_void_p] * 10),
    "b2_sync_committee_messages": (c_int, [c_void_p, c_void_p, c_uint64, c_void_p, c_uint32, c_void_p, c_void_p, c_uint32, c_uint32, c_uint64,
                                           c_void_p] + [c_void_p] * 9),
    # ctx, wire, wire_len, woff, n, position_validator, committee_size, subnet_count, current_slot, domains96, target_aggregators, seven
    # outputs[, stream]
    "b2_sync_contribution_and_proof_intake_dev": (c_int, [c_void_p, c_void_p, c_uint64, c_void_p, c_uint32, c_void_p, c_uint32, c_uint32, c_uint64,
                                                          c_void_p, c_uint32] + [c_void_p] * 8),
    "b2_sync_contribution_and_proof_intake": (c_int, [c_void_p, c_void_p, c_uint64, c_void_p, c_uint32, c_void_p, c_uint32, c_uint32, c_uint64,
                                                      c_void_p, c_uint32] + [c_void_p] * 7),
    "b2_vote_weights_dev": (c_int, [c_void_p, c_void_p, c_void_p]),
    "b2_vote_weights_range_dev": (c_int, [c_void_p, c_uint64, c_uint64, c_void_p, c_void_p]),
    "b2_guard_flags": (c_int, [c_void_p, c_void_p]),
    "b2_gather_probe_dev": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_uint32, c_uint32, c_int, c_void_p, c_void_p]),
    "b2_head_from_votes_dev": (c_int, [c_void_p, c_void_p, c_uint32, c_int32, c_uint64, c_void_p, c_void_p, c_void_p]),
    "b2_tree_size": (c_uint32, [c_void_p]),
    "b2_fc_exchange_export": (c_int, [c_void_p, c_void_p]),
    "b2_fc_exchange_open": (c_int, [c_void_p, c_int, c_int, c_void_p]),
    "b2_get_head_multi": (c_int, [c_void_p, c_uint64, c_uint64, c_uint32, c_int32, c_uint64, c_void_p]),
    "b2_debug_head_clocks": (c_int, [c_void_p, c_void_p]),
    "b2_ssz_validators_load": (c_int, [c_void_p, c_void_p, c_uint64, c_void_p]),
    "b2_ssz_validators_update": (c_int, [c_void_p, c_void_p, c_void_p, c_uint64, c_void_p]),
    "b2_ssz_chunks_root": (c_int, [c_void_p, c_void_p, c_uint64, c_uint32, c_int, c_uint64, c_void_p]),
}


def load():
    """Load the shared library (once) and declare every prototype.  Needs no GPU."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError("%s is missing: build it with `python -m pos_evolution_b200.build` "
                          "(nvcc, sm_90a).  There is no CPU fallback." % LIB_PATH)
    lib = ctypes.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)          # AttributeError if the .so does not export a declared symbol
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib
