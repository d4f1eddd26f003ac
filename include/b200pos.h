/* b200pos.h -- C ABI of libb200pos.so: H100-native attestation aggregation + LMD-GHOST fork choice.
 *
 * Drop-in boundary for the hot path of pos-evolution.md (ethereum/pos-evolution)
 *     process_attestation (:722) -> bls.Aggregate / FastAggregateVerify -> get_head (:1102)
 * The reference is executable Python (pyspec) and has no FFI of its own; the functions below are
 * what a ctypes binding behind the pyspec names would call (INTEGRATION.md shows the stub).
 * Each entry point cites the reference interface it replaces.
 *
 * Conventions
 *   - plain C, no C++/torch types; the caller owns every buffer; the library keeps only the
 *     registry / block-tree / latest-message tables it allocated on the device.
 *   - return value: 0 = ok, negative = B2_E* (environment / argument errors).  Cryptographic
 *     invalidity is DATA (ok_out[i] = 0, seg_status[i] != 0), never an error code.  On error no
 *     output buffer and no device table is modified (pos-evolution.md:1041).  This includes the
 *     table loads: a failed b2_registry_load / b2_tree_load leaves the previous tables in place.
 *   - functions without the _dev suffix take HOST pointers, are synchronous and do their own
 *     host<->device copies.  *_dev functions take DEVICE pointers plus a cudaStream_t (as void*)
 *     and only enqueue work (used by bench.py and by the multi-GPU path, where the u64 vote
 *     weights are all-reduced by NCCL between b2_vote_weights_dev and b2_head_from_votes_dev).
 *     Both forms of an entry point reject the same arguments with the same b2_last_error text;
 *     the host form also checks the contents of its host arrays (offsets, indices, epochs).
 *   - a b2_ctx is bound to one GPU and is not thread-safe (pyspec is single-threaded).
 *   - there is no CPU fallback: b2_init fails with B2_ENODEVICE when no sm_90 (H100) GPU is present.
 */
#ifndef B200POS_H
#define B200POS_H
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct b2_ctx b2_ctx;

enum {
    B2_OK = 0,
    B2_EINVAL = -1,    /* bad argument (null pointer, index out of range, missing table) */
    B2_ECUDA = -2,     /* CUDA runtime error; b2_last_error() has the text */
    B2_ENODEVICE = -3, /* no usable GPU */
    B2_ENOMEM = -4
};

/* status bits written by b2_g1_aggregate (why py_ecc's FastAggregateVerify would return False) */
enum { B2_PK_OK = 0, B2_PK_INVALID_KEY = 1, B2_PK_EMPTY = 2, B2_PK_INFINITY = 4, B2_PK_BAD_INDEX = 8 };

int b2_init(int device, b2_ctx** out);
void b2_destroy(b2_ctx* ctx);
const char* b2_last_error(b2_ctx* ctx);
int b2_sync(b2_ctx* ctx);
/* number of kernels this context has launched so far (bench.py's gpu_launches) */
uint64_t b2_launch_count(b2_ctx* ctx);

/* ---- validator registry: BeaconState.validators[*].{pubkey, effective_balance} (pos-evolution.md:36-45, :354).
 * Decompresses and KeyValidates every pubkey ONCE (py_ecc does it on every FastAggregateVerify call) and
 * keeps 96-byte affine Montgomery records on the device.  flags: bit0 = active at the fork-choice epoch
 * (is_active_validator), bit1 = slashed.  pk_valid_out (may be NULL): 1 = KeyValidate passed. */
int b2_registry_load(b2_ctx* ctx, const uint8_t* pk48, const uint64_t* effective_balance, const uint8_t* flags,
                     uint64_t n_validators, uint8_t* pk_valid_out);
/* bls.KeyValidate (decodable, not infinity, in the r-torsion; eth2spec.utils.bls, used by process_deposit upstream) for n explicit
 * pubkeys; leaves the registry alone. */
int b2_key_validate(b2_ctx* ctx, const uint8_t* pk48, uint64_t n, uint8_t* valid_out);
/* refresh balances / flags only (process_effective_balance_updates, pos-evolution.md:122-133, changes them per epoch) */
int b2_registry_update_balances(b2_ctx* ctx, const uint64_t* effective_balance, const uint8_t* flags, uint64_t n_validators);

/* ---- committees and aggregation bits (get_beacon_committee :729, get_attesting_indices :745):
 * aggregate a has members[off[a] .. off[a+1]) (validator indices, committee order) and bit j of
 * bits[a*bits_stride ...] (little-endian within bytes, SSZ Bitlist order) selects member j. */

/* K2: per aggregate, sum of the selected pubkeys; out48 = compressed G1 (infinity encoding when empty). */
int b2_g1_aggregate(b2_ctx* ctx, const uint32_t* members, const uint32_t* off, const uint8_t* bits, uint32_t bits_stride,
                    uint32_t n_agg, uint8_t* out48, uint8_t* status);

/* bls.Aggregate (eth2spec.utils.bls; named by BASELINE.json, called as get_aggregate_signature upstream), batched:
 * segment s = signatures [seg_off[s], seg_off[s+1]).  seg_status: 0 ok, 1 = a signature is undecodable
 * (py_ecc raises), 2 = empty segment (py_ecc raises).  No subgroup check, as in py_ecc. */
int b2_aggregate(b2_ctx* ctx, const uint8_t* sig96, const uint32_t* seg_off, uint32_t n_seg, uint8_t* out96, int32_t* seg_status);

/* bls.FastAggregateVerify inside is_valid_indexed_attestation (pos-evolution.md:736, :976), batched over
 * aggregates, pubkeys taken from the registry by index.  ok_out[a] in {0,1}; never an error for bad crypto. */
int b2_fast_aggregate_verify(b2_ctx* ctx, const uint32_t* members, const uint32_t* off, const uint8_t* bits, uint32_t bits_stride,
                             const uint8_t* msg32, const uint8_t* sig96, uint32_t n_agg, uint8_t* ok_out);

/* pyspec-literal form: explicit compressed pubkeys, aggregate a uses pk48[pk_off[a] .. pk_off[a+1]).
 * Decompresses + KeyValidates every key on every call (what py_ecc does).  bls.Verify (:165) is the 1-key case. */
int b2_fast_aggregate_verify_pks(b2_ctx* ctx, const uint8_t* pk48, const uint32_t* pk_off, const uint8_t* msg32,
                                 const uint8_t* sig96, uint32_t n_agg, uint8_t* ok_out);

/* bls.AggregateVerify (IETF POP scheme: messages need NOT be distinct), batched.  Set s = pairs [pair_off[s], pair_off[s+1]):
 * (pk48[i], msg32[i]) for each pair, and one signature sig96[s].  ok_out[s] = 1 iff the set is non-empty, every key passes
 * KeyValidate, the signature decodes and lies in G2, and  prod_i e(pk_i, H(m_i)) * e(-g1, S) == 1: n + 1 Miller loops and ONE final
 * exponentiation per set.  Not affected by b2_set_verify_mode (always the exact per-set equation). */
int b2_aggregate_verify_pks(b2_ctx* ctx, const uint8_t* pk48, const uint8_t* msg32, const uint32_t* pair_off, const uint8_t* sig96,
                            uint32_t n_sets, uint8_t* ok_out);
/* the same with the signers taken from the registry by index (keys validated once at b2_registry_load); a signer index
 * >= n_validators is B2_EINVAL */
int b2_aggregate_verify(b2_ctx* ctx, const uint32_t* signer, const uint8_t* msg32, const uint32_t* pair_off, const uint8_t* sig96,
                        uint32_t n_sets, uint8_t* ok_out);
/* bls.AggregatePKs (py_ecc _AggregatePKs), batched: segment s = pk48[off[s] .. off[s+1]) -> compressed sum (the infinity encoding
 * when the keys cancel); status = B2_PK_* bits of b2_g1_aggregate (B2_PK_INVALID_KEY, B2_PK_EMPTY; B2_PK_INFINITY alone is a valid result) */
int b2_aggregate_pks(b2_ctx* ctx, const uint8_t* pk48, const uint32_t* off, uint32_t n_seg, uint8_t* out48, uint8_t* status);

/* ---- sync committees (pos-evolution.md:371-372, :540-590; Altair process_sync_aggregate): n_committees tables of committee_size keys
 * (1 <= committee_size <= 1024), pk48 = committee after committee.  Decodes + KeyValidates every key and sums each committee's valid
 * keys ONCE; valid_out (may be NULL): 1 = KeyValidate passed, per key.  Replaces the previously loaded committees only on success. */
int b2_sync_committee_load(b2_ctx* ctx, const uint8_t* pk48, uint32_t committee_size, uint32_t n_committees, uint8_t* valid_out);
/* eth_fast_aggregate_verify (Altair bls helper) of block i: participants = the keys of committee committee_idx[i] whose bit is set in
 * bits[i * ceil(committee_size/8) ...] (SSZ Bitvector order; bits past committee_size are ignored); msg32 = signing root.  ok_out[i] in
 * {0,1}: FastAggregateVerify over the participants' keys, except that no participant accepts exactly the G2 infinity signature
 * (0xc0 then 95 zero bytes).  The aggregate key is the sum of the participants or the committee sum minus the non-participants,
 * whichever needs fewer additions.  pk48_out (may be NULL): the compressed sum of the participants' valid keys per block.
 * Needs no registry; a committee index >= n_committees, or no loaded committee, is B2_EINVAL.  b2_set_verify_mode applies. */
int b2_sync_aggregate_verify(b2_ctx* ctx, const uint32_t* committee_idx, const uint8_t* bits, const uint8_t* msg32, const uint8_t* sig96,
                             uint32_t n, uint8_t* ok_out, uint8_t* pk48_out);
/* the same on device arrays (asynchronous on `stream`): a committee index >= n_committees fails only its own block and sets
 * B2_GUARD_BAD_INDEX */
int b2_sync_aggregate_verify_dev(b2_ctx* ctx, const uint32_t* d_committee_idx, const uint8_t* d_bits, const uint8_t* d_msg32,
                                 const uint8_t* d_sig96, uint32_t n, uint8_t* d_ok_out, uint8_t* d_pk48_out, void* stream);

/* bls.SkToPk / bls.Sign, batched (sk = 8 little-endian u32 limbs, 0 < sk < r).  Signature i = sk[i] * H(msg[msg_idx[i]]). */
int b2_sk_to_pk(b2_ctx* ctx, const uint32_t* sk8, uint64_t n, uint8_t* pk48_out);
int b2_sign(b2_ctx* ctx, const uint32_t* sk8, const uint32_t* msg_idx, uint64_t n, const uint8_t* msg32, uint32_t n_msg,
            uint8_t* sig96_out);
/* H(m) compressed, for tests (hash_to_G2 with the POP ciphersuite tag) */
int b2_hash_to_g2(b2_ctx* ctx, const uint8_t* msg32, uint32_t n_msg, uint8_t* out96);

/* `hash` of the spec (SHA-256; pos-evolution.md:486, :522, :525), batched over n messages of msg_len bytes each */
int b2_sha256_batch(b2_ctx* ctx, const uint8_t* msgs, uint32_t msg_len, uint64_t n, uint8_t* out32);

/* SSZ wire form of n Attestations (pos-evolution.md:714-717, AttestationData :689-697): each is
 *   [u32 LE offset of aggregation_bits = 228][AttestationData 128 B][signature 96 B][Bitlist bytes, length given by the delimiter bit].
 * wire = the encodings back to back, woff u32[n+1] their byte offsets.  Outputs per attestation: the bit row (delimiter removed,
 * zero padded to bits_stride bytes -- the form b2_fast_aggregate_verify / b2_latest_messages_update take), its bit length, the
 * 128-byte AttestationData record (the input of b2_signing_roots) and the signature.
 * status_out: 0 ok; 1 malformed container; 2 empty Bitlist / no delimiter; 3 longer than max_bits (MAX_VALIDATORS_PER_COMMITTEE)
 * or than bits_stride allows.  A rejected attestation yields zero rows: malformed input is data, not an error. */
int b2_attestations_decode(b2_ctx* ctx, const uint8_t* wire, const uint32_t* woff, uint32_t n, uint32_t bits_stride, uint32_t max_bits,
                           uint8_t* bits_out, uint32_t* bit_len_out, uint8_t* data128_out, uint8_t* sig96_out, int32_t* status_out);

/* compute_signing_root(AttestationData, domain) (pattern of pos-evolution.md:163; containers :689-697, :219-221) for n attestations:
 * data128 = the 128-byte SSZ serialisation of each AttestationData; domain32 = one 32-byte domain for the batch, or one per
 * attestation when per_attestation_domain != 0.  SSZ merkleization (10 SHA-256 per attestation) runs on the GPU. */
int b2_signing_roots(b2_ctx* ctx, const uint8_t* data128, const uint8_t* domain32, int per_attestation_domain, uint32_t n, uint8_t* out32);

/* ---- committees: compute_committee / compute_shuffled_index (pos-evolution.md:495-534) for a whole epoch.
 * members_out[i] = active[compute_shuffled_index(i, n_active, seed)] (active == NULL: identity), so committee k of
 * `count` is members_out[n*k/count .. n*(k+1)/count).  SHA-256 and the swap-or-not rounds run on the GPU. */
int b2_shuffle_committees(b2_ctx* ctx, const uint8_t* seed32, const uint32_t* active, uint32_t n_active, uint32_t rounds,
                          uint32_t* members_out);
int b2_shuffle_committees_dev(b2_ctx* ctx, const uint8_t* d_seed32, const uint32_t* d_active, uint32_t n_active, uint32_t rounds,
                              uint32_t* d_members_out, void* stream);

/* ---- fork choice --------------------------------------------------------------------------------
 * Store.latest_messages (pos-evolution.md:901) lives on the device as (epoch, block index) per validator. */
int b2_latest_messages_reset(b2_ctx* ctx);
/* bulk load: has_msg[v] != 0 -> (epoch[v], block_idx[v]); equivocating[v] != 0 -> Store.equivocating_indices (:897) */
int b2_latest_messages_load(b2_ctx* ctx, const uint64_t* epoch, const uint32_t* block_idx, const uint8_t* has_msg,
                            const uint8_t* equivocating, uint64_t n_validators);
int b2_latest_messages_read(b2_ctx* ctx, uint64_t* epoch, uint32_t* block_idx, uint8_t* has_msg, uint64_t n_validators);
/* update_latest_messages (pos-evolution.md:1435-1441) for a batch of attestations in list order:
 * for each accepted aggregate a (accept[a] != 0, or accept == NULL) and each selected member i not equivocating:
 * set (target_epoch[a], block_idx[a]) iff i has no message or target_epoch[a] > stored epoch.  Order-exact. */
int b2_latest_messages_update(b2_ctx* ctx, const uint32_t* members, const uint32_t* off, const uint8_t* bits, uint32_t bits_stride,
                              const uint64_t* target_epoch, const uint32_t* block_idx, const uint8_t* accept, uint32_t n_agg);

/* ---- participation flags and proposer-reward numerators: the bookkeeping loop of process_attestation (pos-evolution.md:738-754).
 * `which`: 0 = state.current_epoch_participation, 1 = previous.  For a batch of attestations in list order, each accepted
 * attestation a sets, for every selected member, the flags of flag_mask[a] (bit f = participation flag index f) that are not set
 * yet, and numerator_out[a] receives sum get_base_reward(index) * PARTICIPATION_FLAG_WEIGHTS[f] over the flags IT set
 * (get_base_reward = effective_balance / increment * base_reward_per_increment).  Order-exact for the whole batch. */
int b2_participation_load(b2_ctx* ctx, int which, const uint8_t* participation, uint64_t n_validators);
int b2_participation_read(b2_ctx* ctx, int which, uint8_t* participation_out, uint64_t n_validators);
int b2_participation_update(b2_ctx* ctx, int which, const uint32_t* members, const uint32_t* off, const uint8_t* bits, uint32_t bits_stride,
                            const uint8_t* flag_mask, const uint8_t* accept, uint32_t n_agg, uint64_t effective_balance_increment,
                            uint64_t base_reward_per_increment, uint64_t* numerator_out);

/* ---- FFG balance sums: the inputs of weigh_justification_and_finalization (pos-evolution.md:793-803, :817-837).
 * out4[0] = get_total_active_balance (sum of effective balances, registry flag bit0 = active in the current epoch),
 * out4[1] / out4[2] = get_total_balance(get_unslashed_participating_indices(state, flag_index, current / previous epoch)): validators
 *           that are active in that epoch (flag bit0 / bit2), not slashed (bit1) and carry `flag_index` in the participation table
 *           `which` = 0 / 1 (b2_participation_load; a table that was never loaded counts as all-zero),
 * out4[3] = total active AND unslashed balance (the essay's prose reading of get_total_active_balance, :809).
 * Raw sums: the caller applies max(EFFECTIVE_BALANCE_INCREMENT, .) as get_total_balance does. */
int b2_ffg_balances(b2_ctx* ctx, uint32_t flag_index, uint64_t* out4);

/* ---- fork-choice variants (pos-evolution.md:1411-1413, :1447-1461, :1549-1596):
 * b2_set_fork_choice_params: votes whose epoch is < min_vote_epoch do not count (vote expiry of the Goldfish / RLMD-GHOST family;
 *   0 = plain LMD-GHOST); exclude_slashed != 0 selects the v1.3 get_weight rule (slashed validators, registry flag bit1, do not count).
 * b2_on_attester_slashing: the validators present in BOTH sorted index lists become equivocating (Store.equivocating_indices)
 *   and stop counting; validity of the slashing itself (:1453-1457) is the caller's job. */
int b2_set_fork_choice_params(b2_ctx* ctx, uint64_t min_vote_epoch, int exclude_slashed);
/* How bls.FastAggregateVerify (is_valid_indexed_attestation, pos-evolution.md:736/:976) is evaluated for a BATCH of aggregates:
 *   mode 0 (default): e(PK_a, H(m_a)) * e(-g1, S_a) == 1 for every aggregate a (two Miller loops + one final exponentiation each);
 *   mode 1: random-linear-combination batches -- per group of 32 aggregates ONE equation
 *           prod_a e([r_a] PK_a, H(m_a)) * e(-g1, sum_a [r_a] S_a) == 1, r_a = 64-bit scalars derived by SHA-256 from `seed32`
 *           (the verifier's secret: pass fresh randomness), i.e. one Miller loop per aggregate plus one Miller loop and one final
 *           exponentiation per group; the members of a group whose equation fails are then verified one by one, so ok_out is
 *           the mode-0 vector (a wrong accept needs a 2^-63 coincidence).  Less work, longer critical path: for bulk verification.
 * Synchronises the device.  Applies to every FastAggregateVerify / epoch entry point of the context. */
int b2_set_verify_mode(b2_ctx* ctx, int mode, const uint8_t* seed32);
int b2_on_attester_slashing(b2_ctx* ctx, const uint32_t* indices_1, uint32_t n1, const uint32_t* indices_2, uint32_t n2);

/* ---- slasher: FIND the slashable attestations (is_slashable_attestation_data, pos-evolution.md:1128-1143: double vote, surround vote)
 * among everything that streams through, so that an AttesterSlashing (:1160-1162, on_attester_slashing :1447-1461) can be produced.
 * A slasher is a device-resident history of n_validators validators over a ring of history_epochs (H) epochs with a current epoch `cur`
 * that only moves forward; the window is low = max(0, cur - H + 1) .. cur.  It is independent of the registry; a context that never
 * calls b2_slasher_init allocates nothing.  Memory: 6 * n_validators * H + 32 * H * max_attestations_per_target bytes; the byte count
 * is compared with the free device memory first, and B2_ENOMEM is returned without trying the allocation when it does not fit.  A
 * failed init leaves the context, and a previously initialised slasher, as they were.  H, max_attestations_per_target <= 65535. */
int b2_slasher_init(b2_ctx* ctx, uint64_t n_validators, uint32_t history_epochs, uint32_t max_attestations_per_target, uint64_t current_epoch);
/* The same for the validators [v_begin, v_end) of n_validators only (0 <= v_begin < v_end <= n_validators, else B2_EINVAL): one rank's
 * share of a registry sharded by validator range.  Memory 6 * (v_end - v_begin) * H + 32 * H * max_attestations_per_target + 4 * H bytes,
 * compared with the free device memory as above.  Updates take the whole batch: a member index >= n_validators still sets
 * B2_GUARD_BAD_INDEX (device form) or is B2_EINVAL (host form); a valid member outside [v_begin, v_end) is skipped silently (kind 0,
 * conflict targets 0xffffffff, not counted in n_flagged).  Statuses, ids, column counts and the root log do not depend on the range, so
 * slashers over the ranges of a partition fed the same batches stay consistent, and the union of their kind vectors is the vector of
 * one slasher over all validators.  b2_slasher_init is b2_slasher_init_range(0, n_validators). */
int b2_slasher_init_range(b2_ctx* ctx, uint64_t n_validators, uint64_t v_begin, uint64_t v_end, uint32_t history_epochs,
                          uint32_t max_attestations_per_target, uint64_t current_epoch);
int b2_slasher_free(b2_ctx* ctx); /* also done by b2_destroy */
/* move the current epoch forward (a lower one, or one that does not fit 32 bits, is B2_EINVAL and changes nothing); the columns of the
 * new epochs start empty.  Synchronises the device. */
int b2_slasher_advance(b2_ctx* ctx, uint64_t current_epoch);
/* The same without synchronising: the column reset is enqueued on `stream` and the window moves at enqueue time, so every update
 * enqueued after this call sees the new window and must be stream-ordered after the reset by the caller (same stream, or an event). */
int b2_slasher_advance_dev(b2_ctx* ctx, uint64_t current_epoch, void* stream);
/* Offer n_agg aggregates (members / off / bits as above; source_epoch, target_epoch = data.source.epoch, data.target.epoch;
 * data_root32 = hash_tree_root(AttestationData)).  Aggregate a is ACCEPTED iff accept[a] != 0 (or accept == NULL), s <= t <= cur,
 * s >= low and fewer than max_attestations_per_target aggregates with target t have been accepted; otherwise att_status_out[a] =
 * B2_SLASHER_* says why and it neither checks nor records anything.  For every selected member v of an accepted aggregate (s, t),
 * kind_out (u8[off[n_agg]], parallel to members; 0 for clear bits and unaccepted rows) is evaluated against EVERY attestation by v
 * accepted so far, the other aggregates of this call included, whatever their position (:1128-1143):
 *   B2_SLASHABLE_DOUBLE      the first accepted attestation by v with target t (earliest call, then lowest position) has another root;
 *   B2_SLASHABLE_SURROUNDS   some accepted attestation by v has source > s and target < t; conflict_target_out[i][0] = the smallest such target;
 *   B2_SLASHABLE_SURROUNDED  some accepted attestation by v has source < s and target > t; conflict_target_out[i][1] = the largest such target
 * (conflict_target_out u32[off[n_agg]][2], may be NULL; 0xffffffff where the bit is clear).  Detection is exact against everything ever
 * accepted, not only what is still inside the window.  n_flagged_out = number of member slots with kind != 0. */
enum { B2_SLASHER_OK = 0, B2_SLASHER_NOT_ACCEPTED = 1, B2_SLASHER_SOURCE_AFTER_TARGET = 2, B2_SLASHER_TARGET_AHEAD = 3,
       B2_SLASHER_SOURCE_EXPIRED = 4, B2_SLASHER_COLUMN_FULL = 5, B2_SLASHER_BAD_ROW = 6 /* device form only */ };
enum { B2_SLASHABLE_DOUBLE = 1, B2_SLASHABLE_SURROUNDS = 2, B2_SLASHABLE_SURROUNDED = 4 };
int b2_slasher_update(b2_ctx* ctx, const uint32_t* members, const uint32_t* off, const uint8_t* bits, uint32_t bits_stride,
                      const uint64_t* source_epoch, const uint64_t* target_epoch, const uint8_t* data_root32, const uint8_t* accept, uint32_t n_agg,
                      int32_t* att_status_out, uint8_t* kind_out, uint32_t* conflict_target_out, uint32_t* n_flagged_out);
/* the same on device arrays (asynchronous on `stream`; the arrays b2_epoch_tail_dev / b2_latest_messages_update_dev take, with the
 * verdict bytes as d_accept, so it chains after b2_epoch_wait_dev).  Self-guarding: a malformed offsets row is B2_SLASHER_BAD_ROW and
 * its member slots are not written (B2_GUARD_BAD_ROW); a member index >= n_validators is skipped, its kind stays 0
 * (B2_GUARD_BAD_INDEX); an epoch that does not fit 32 bits sets B2_GUARD_BAD_EPOCH and the row is refused by status 2 or 3. */
int b2_slasher_update_dev(b2_ctx* ctx, const uint32_t* d_members, const uint32_t* d_off, const uint8_t* d_bits, uint32_t bits_stride,
                          const uint64_t* d_source_epoch, const uint64_t* d_target_epoch, const uint8_t* d_data_root32, const uint8_t* d_accept,
                          uint32_t n_agg, int32_t* d_att_status_out, uint8_t* d_kind_out, uint32_t* d_conflict_target_out,
                          uint32_t* d_n_flagged_out, void* stream);

/* ---- equivocation discounting (pos-evolution.md:1405-1461): what the slasher found stops counting in the fork choice.
 * b2_slasher_discount_dev: for every member slot i < n_slots with d_kind[i] != 0 (the d_kind_out of a b2_slasher_update_dev, members
 *   parallel to it), validator d_members[i] joins Store.equivocating_indices -- what on_attester_slashing (:1447-1461) adds for every
 *   AttesterSlashing formable from two accepted aggregates, whose attesting indices intersect in exactly the flagged validators.  From
 *   then on the validator neither moves its latest message (b2_latest_messages_update*, :1435-1441) nor counts in any get_head form (:1411).
 *   d_new_out[i] = 1 for exactly one slot of every validator this call newly marked (0 where it was marked before, by this call's other
 *   slots or earlier: b2_on_attester_slashing, b2_latest_messages_load, an earlier discount), d_n_new_out = how many.  Only validators of
 *   the slasher's range (b2_slasher_init_range) and of the registry are marked.  Asynchronous on `stream`; the tables are never un-marked
 *   (b2_registry_load and b2_latest_messages_load/_reset replace them).  Epoch tails (b2_epoch_tail_dev, b2_epoch_dev) enqueued after this
 *   call apply their latest messages only after it: enqueue the discount of epoch k before the tail of epoch k+1.
 *   B2_EINVAL, with nothing enqueued, on bad arguments, no registry or no slasher. */
int b2_slasher_discount_dev(b2_ctx* ctx, const uint32_t* d_members, const uint8_t* d_kind, uint64_t n_slots, uint8_t* d_new_out,
                            uint32_t* d_n_new_out, void* stream);
/* the same on host arrays (returns when done) */
int b2_slasher_discount(b2_ctx* ctx, const uint32_t* members, const uint8_t* kind, uint64_t n_slots, uint8_t* new_out, uint32_t* n_new_out);
/* Store.equivocating_indices as u8[n_validators] (nonzero = equivocating), after every mark enqueued so far (:1405-1461) */
int b2_equivocating_read(b2_ctx* ctx, uint8_t* out, uint64_t n_validators);
/* Sharded registries (pos-evolution.md:1405-1461): rank g discounts the validators of its slasher range only, so the ranks' replicas of
 * the table are brought together by exchanging range slices.  _slice_dev copies the table's bytes [v_begin, v_end) to d_out;
 * _merge_dev ORs d_table[0 .. v_end - v_begin) into them.  Both asynchronous on `stream`; a merge orders later epoch tails like a discount.
 * B2_EINVAL unless v_begin < v_end <= n_validators of the loaded registry. */
int b2_equivocating_slice_dev(b2_ctx* ctx, uint64_t v_begin, uint64_t v_end, uint8_t* d_out, void* stream);
int b2_equivocating_merge_dev(b2_ctx* ctx, uint64_t v_begin, uint64_t v_end, const uint8_t* d_table, void* stream);

/* ---- block packing: BeaconBlockBody.attestations (List[Attestation, MAX_ATTESTATIONS], pos-evolution.md:639; "well-packed aggregate
 * attestations", :659) chosen from a pool, the proposing-side counterpart of process_attestation (:722-754).
 * Committee k = members[committee_off[k] .. committee_off[k+1]) with participation table committee_table[k] (0 current, 1 previous; the
 * tables of b2_participation_load, a table never loaded counts as all-zero).  Candidate c (pool order) = committee cand_committee[c],
 * data id cand_data[c] (< n_cand; equal ids = the same AttestationData, so the same committee and mask), bit row
 * bits[c * bits_stride ...] (bits at or past the committee size are ignored), flag mask cand_flag_mask[c] (bit f = participation flag f;
 * bits 3..7 ignored) and signature sig96[c].  Precondition: the committees of one table are pairwise disjoint and repeat no member.
 *   1. a candidate whose signature does not decode is excluded (cand_status 1; no subgroup check, as bls.Aggregate);
 *   2. fold, per data id in pool order: a candidate joins the first folded aggregate of its data id (creation order) whose union row is
 *      disjoint from its row, else opens a new one; folded aggregates are numbered by the pool position of their first constituent;
 *   3. gain of a folded aggregate against participation P = sum over its members v and flags f of its mask not in P[v] of
 *      (eff[v] / effective_balance_increment) * base_reward_per_increment * (14, 26, 14)[f] -- the numerator b2_participation_update credits;
 *   4. up to max_out times, pick the largest gain > 0 (tie: lowest committee, then lowest folded number) and set its flags in a private
 *      copy of P.
 * Outputs in pick order: *n_out; per output committee, data id, union bit row (bits_stride bytes, zero padded), the gain as a u64
 * numerator, constituents out_src[out_src_off[o] .. out_src_off[o+1]) in pool order, and the signature (bls.Aggregate of the
 * constituents; one constituent: its bytes unchanged).  Slots past n_out are zero; out_src_off has max_out + 1 entries (past n_out they
 * repeat the total); out_src holds n_cand entries (zero past the total).  cand_status u8[n_cand]: 0 folded, 1 undecodable.  Neither the
 * registry nor the participation tables change.  Applying the outputs in order with b2_participation_update returns the numerators.
 * B2_EINVAL (nothing written): no registry, max_out == 0, bits_stride == 0 or > 256, a committee larger than 8 * bits_stride, a member
 * index >= n_validators, overlapping committees of one table, a table byte > 1, cand_committee >= n_committees, a data id >= n_cand or
 * with two committees or two masks. */
int b2_pack_attestations(b2_ctx* ctx, const uint32_t* members, const uint32_t* committee_off, const uint8_t* committee_table, uint32_t n_committees,
                         const uint32_t* cand_committee, const uint32_t* cand_data, const uint8_t* cand_flag_mask, const uint8_t* bits, uint32_t bits_stride,
                         const uint8_t* sig96, uint32_t n_cand, uint32_t max_out, uint64_t effective_balance_increment, uint64_t base_reward_per_increment,
                         uint32_t* n_out, uint32_t* out_committee, uint32_t* out_data, uint8_t* out_bits, uint8_t* out_sig96, uint64_t* out_numerator,
                         uint32_t* out_src_off, uint32_t* out_src, uint8_t* cand_status);
/* the same on device arrays, asynchronous on `stream` (d_n_out is written on the device).  Self-guarding: a candidate committee index
 * >= n_committees excludes the candidate (cand_status 2, B2_GUARD_BAD_INDEX); a member index >= n_validators earns nothing
 * (B2_GUARD_BAD_INDEX); overlapping committees of one table, a malformed committee row (also B2_GUARD_BAD_ROW), a table byte > 1, or a
 * data id >= n_cand or with two committees or masks set B2_GUARD_BAD_POOL and the call selects nothing (n_out = 0). */
int b2_pack_attestations_dev(b2_ctx* ctx, const uint32_t* d_members, const uint32_t* d_committee_off, const uint8_t* d_committee_table,
                             uint32_t n_committees, const uint32_t* d_cand_committee, const uint32_t* d_cand_data, const uint8_t* d_cand_flag_mask,
                             const uint8_t* d_bits, uint32_t bits_stride, const uint8_t* d_sig96, uint32_t n_cand, uint32_t max_out,
                             uint64_t effective_balance_increment, uint64_t base_reward_per_increment, uint32_t* d_n_out, uint32_t* d_out_committee,
                             uint32_t* d_out_data, uint8_t* d_out_bits, uint8_t* d_out_sig96, uint64_t* d_out_numerator, uint32_t* d_out_src_off,
                             uint32_t* d_out_src, uint8_t* d_cand_status, void* stream);

/* Store.blocks (pos-evolution.md:898) as arrays in topological order (parent[b] < b, parent[0] ignored; block 0 =
 * store.justified_checkpoint.root).  leaf_viable[b]: the get_filtered_block_tree leaf test (:1104, prose :1121-1124). */
int b2_tree_load(b2_ctx* ctx, const uint32_t* parent, const uint64_t* slot, const uint8_t* root32, const uint8_t* leaf_viable,
                 uint32_t n_blocks);
/* get_latest_attesting_balance == get_weight (called at pos-evolution.md:1116) for EVERY block; boost_idx < 0: no boost */
int b2_get_weights(b2_ctx* ctx, int32_t boost_idx, uint64_t boost_score, uint64_t* weight_out);
/* get_head (pos-evolution.md:1102-1116): index of the head block */
int b2_get_head(b2_ctx* ctx, uint32_t justified_idx, int32_t boost_idx, uint64_t boost_score, uint32_t* head_idx_out);
/* ---- changing the loaded tree on the device, without a reload.  After any sequence of these calls the context behaves exactly like
 * b2_tree_load of the resulting arrays (parent, root, leaf_viable in id order): the same kernel form, weights, heads and tie-breaks.
 * Each call is synchronous.  A rejected call (B2_EINVAL: no tree loaded, k == 0, a parent >= its own id, a prune root or a viability
 * index >= n) changes nothing.  A change of size needs b2_fc_exchange_export / _open again before b2_get_head_multi.
 *   b2_tree_add        on_block adds a block to store.blocks (pos-evolution.md:1015-1018): appends k blocks, which take ids n .. n+k-1;
 *                      parent[j] < n + j, so a batch may parent within itself.  The arrays are those of b2_tree_load.
 *   b2_tree_prune      the finalized checkpoint moves (:1033-1036): keeps the subtree of new_root, which becomes id 0; the kept blocks
 *                      keep their order (parents still precede children).  map_out (the old n entries) receives map[old] = new id, or
 *                      0xFFFFFFFF for a dropped block.  Every validator's latest-message block is re-mapped through it; the message
 *                      epochs and equivocation flags are untouched, and a vote for a dropped block counts nowhere.  The re-map runs on
 *                      the context's own stream: device-pointer work the caller queued on its streams that reads or writes the
 *                      latest messages or a vote vector (b2_latest_messages_update_dev, b2_vote_weights_*dev, b2_epoch_*_dev) must be
 *                      complete before the call.
 *   b2_tree_set_viable the get_filtered_block_tree leaf test (:1104): sets the viability byte of blocks idx[0..k) (only leaves' bytes
 *                      matter, as in b2_tree_load; a repeated index keeps its last value). */
int b2_tree_add(b2_ctx* ctx, const uint32_t* parent, const uint64_t* slot, const uint8_t* root32, const uint8_t* leaf_viable, uint32_t k);
int b2_tree_prune(b2_ctx* ctx, uint32_t new_root, uint32_t* map_out);
int b2_tree_set_viable(b2_ctx* ctx, const uint32_t* idx, const uint8_t* viable, uint32_t k);

/* ---- device-pointer entry points (asynchronous on `stream`) ------------------------------------------------------
 * The host cannot read what device pointers point to, so the checks the host entry points make before touching anything
 * (check_batch: monotone offsets, rows no longer than the bit row, member indices inside the registry, epochs < 2^32 - 1) are made by
 * the kernels themselves: an offending aggregate is skipped -- it fails verification (status B2_PK_BAD_INDEX), joins no LMD update,
 * its segment is reported undecodable -- nothing is read or written out of bounds, and the event is recorded in a guard word.
 * Precondition that cannot be checked on the device: off[n_agg] <= length of the members array.
 * b2_guard_flags: synchronises, returns and clears that word (bit0 member index >= n_validators, bit1 malformed offsets row,
 * bit2 target epoch does not fit 32 bits, bit3 a pool b2_pack_attestations_dev refused). */
enum { B2_GUARD_BAD_INDEX = 1, B2_GUARD_BAD_ROW = 2, B2_GUARD_BAD_EPOCH = 4, B2_GUARD_BAD_POOL = 8 };
int b2_guard_flags(b2_ctx* ctx, uint32_t* flags_out);
int b2_aggregate_dev(b2_ctx* ctx, const uint8_t* d_sig96, const uint32_t* d_seg_off, uint32_t n_seg, uint64_t n_sig, uint8_t* d_out96,
                     int32_t* d_seg_status, void* stream);
int b2_fast_aggregate_verify_dev(b2_ctx* ctx, const uint32_t* d_members, const uint32_t* d_off, const uint8_t* d_bits,
                                 uint32_t bits_stride, const uint8_t* d_msg32, const uint8_t* d_sig96, uint32_t n_agg,
                                 uint8_t* d_ok_out, void* stream);
/* b2_aggregate_verify on device arrays: d_signer / d_msg32 hold n_pairs entries.  A signer index >= n_validators fails only its own set
 * (B2_GUARD_BAD_INDEX).  Malformed offsets -- d_pair_off[0] != 0, a decreasing pair, or d_pair_off[n_sets] > n_pairs -- fail EVERY set
 * of the call (the item -> set mapping needs monotone offsets) and set B2_GUARD_BAD_ROW; nothing is read out of bounds either way. */
int b2_aggregate_verify_dev(b2_ctx* ctx, const uint32_t* d_signer, const uint8_t* d_msg32, const uint32_t* d_pair_off, uint64_t n_pairs,
                            const uint8_t* d_sig96, uint32_t n_sets, uint8_t* d_ok_out, void* stream);
/* The gather stage of K2 alone, for measurement (north_star: ">= 60 % of HBM-read roofline on the pubkey gather"): for every aggregate
 * the XOR of the 24 record words of each selected member's pubkey record (get_attesting_indices + the pubkey list of
 * is_valid_indexed_attestation, pos-evolution.md:736/:745, without the additions).  form 1 = TMA-staged (cp.async.bulk -> shared
 * memory -> 128-bit LDS, the path b2_fast_aggregate_verify uses), form 0 = plain 128-bit global loads.  Both give the same words. */
int b2_gather_probe_dev(b2_ctx* ctx, const uint32_t* d_members, const uint32_t* d_off, const uint8_t* d_bits, uint32_t bits_stride,
                        uint32_t n_agg, int form, uint32_t* d_checksum_out, void* stream);
/* One epoch of this rank in one call: bls.Aggregate per committee (segment a = signatures [off[a], off[a+1]), one per member, in
 * committee order) -> FastAggregateVerify of the aggregates -> update_latest_messages for the accepted ones.  The pubkey/hash half
 * of the verification is overlapped with the signature decompression on side streams. */
int b2_epoch_dev(b2_ctx* ctx, const uint8_t* d_sig96, const uint32_t* d_members, const uint32_t* d_off, const uint8_t* d_bits,
                 uint32_t bits_stride, const uint8_t* d_msg32, const uint64_t* d_target_epoch, const uint32_t* d_block_idx, uint32_t n_agg,
                 uint64_t n_sig, uint8_t* d_agg_sig96, int32_t* d_agg_status, uint8_t* d_ok_out, void* stream);
/* Software-pipelined form of b2_epoch_dev.  Epoch k uses slot = k mod depth, depth <= B2_EPOCH_SLOTS:
 *   b2_epoch_start_dev(slot)  on `stream`: forks the pubkey/hash half, decompresses and segment-sums the signatures (waits until
 *                             the slot's previous tail has drained);
 *   b2_epoch_tail_dev(slot)   on the slot's own high-priority stream: inversion + compress, subgroup check, second Miller loop,
 *                             final exponentiation, update_latest_messages (applied in epoch order).  Its outputs (aggregate
 *                             signatures, verdicts, the LMD table) are valid for a stream only after b2_epoch_wait_dev(slot, it).
 *                             d_target_epoch == d_block_idx == NULL: no LMD update in the tail -- the form of a SHARDED epoch (one
 *                             validator set, committees split over ranks by slot, pos-evolution.md:455), whose caller all-gathers
 *                             the verdicts and then applies b2_latest_messages_update_dev for ALL aggregates on every rank;
 *   fork choice of epoch k    b2_epoch_wait_dev(slot, s); b2_vote_weights_dev(s); all-reduce; b2_head_from_votes_dev(s) -- enqueue it
 *                             before the tail of epoch k+1, whose LMD update waits for the vote scatter issued before it.
 * The latency-bound tails of epochs k, k-1, .. thereby overlap with each other and with the grid-filling signature decompression of
 * epoch k+1: under that contention one tail takes longer than one decompression, so depth 3 is what keeps the multiply pipe busy. */
#define B2_EPOCH_SLOTS 16
int b2_epoch_start_dev(b2_ctx* ctx, int slot, const uint8_t* d_sig96, const uint32_t* d_members, const uint32_t* d_off, const uint8_t* d_bits,
                       uint32_t bits_stride, const uint8_t* d_msg32, uint32_t n_agg, uint64_t n_sig, int32_t* d_agg_status, void* stream);
int b2_epoch_tail_dev(b2_ctx* ctx, int slot, const uint32_t* d_members, const uint32_t* d_off, const uint8_t* d_bits, uint32_t bits_stride,
                      const uint64_t* d_target_epoch, const uint32_t* d_block_idx, uint32_t n_agg, uint8_t* d_agg_sig96, int32_t* d_agg_status,
                      uint8_t* d_ok_out);
int b2_epoch_wait_dev(b2_ctx* ctx, int slot, void* stream);
/* Which form of the pairing kernels (K5/K6) b2_epoch_start_dev / b2_epoch_tail_dev enqueue from now on: 0 = thread per aggregate
 * (fewest instructions: right while further epochs keep the chip busy), 1 = three lanes per pairing (shortest critical path: right for
 * the last epochs of a batch, whose tails drain with nothing left to overlap).  The synchronous entry points always use form 1. */
int b2_epoch_set_pairing_form(b2_ctx* ctx, int form);
/* ---- vote form of an epoch: committees whose members signed different AttestationData (pos-evolution.md:714-717 Attestation, :722-754
 * process_attestation; a split committee is what proposer boost and equivocation discounting exist to defeat).  Committee c has members
 * d_members[d_off[c] .. d_off[c+1]) and the vote ids [d_vote_off[c], d_vote_off[c+1]) (strictly increasing, d_vote_off[0] = 0,
 * d_vote_off[n_committees] = n_votes: every committee has at least one id, a committee where nobody attested one placeholder).
 * d_vote[j] = the id member j signed, or 0xFFFFFFFF if it did not attest.  b2_votes_group_dev stable-sorts each committee's positions
 * by vote, one CTA per committee, keeping committee order within a vote; non-attesters go last and belong to the committee's last vote.
 * Outputs, the arrays b2_epoch_dev / b2_epoch_start_dev / _tail_dev, b2_latest_messages_update_dev (update_latest_messages, :1435-1441)
 * and the slasher take with n_agg = n_votes:
 *   d_members_out u32[n_sig], d_pos_out u32[n_sig]  the grouped members and the committee position each came from;
 *   d_seg_off u32[n_votes+1]                         vote v = grouped slots [d_seg_off[v], d_seg_off[v+1]), inside its committee's
 *                                                    range: d_seg_off[d_vote_off[c]] = d_off[c], d_seg_off[n_votes] = d_off[n_committees];
 *   d_bits_out u8[n_votes][bits_stride]              the first count_v bits set (count_v = the vote's attesters);
 *   d_agg_bits_out u8[n_votes][bits_stride]          the vote's aggregation_bits over committee positions;
 *   d_sig96_out                                      the signatures of committees [c_begin, c_end) grouped (index 0 = d_off[c_begin],
 *                                                    as d_sig96), a non-attester's slot replaced by the infinity encoding 0xc0 || 0^95;
 *   d_seg_off_loc (may be NULL) u32[...]             d_seg_off of the votes [d_vote_off[c_begin], d_vote_off[c_end)] minus d_off[c_begin]:
 *                                                    the offsets of one rank's committees over its own signatures.
 * With one vote per committee and everyone attesting the outputs equal the inputs.  Self-guarding: an id outside its committee's
 * range (not 0xFFFFFFFF) counts as not attesting (B2_GUARD_BAD_INDEX); a malformed d_vote_off empties every vote of the call, and a
 * committee row that is reversed, ends past n_sig, exceeds 8 * bits_stride members or votes, or (within [c_begin, c_end)) leaves the
 * range's signatures empties that committee's votes (B2_GUARD_BAD_ROW); nothing is read or written out of bounds.  b2_votes_empty_dev
 * then makes every vote without attester (bit 0 of its d_bits_out row clear) read like an empty segment after the epoch: status 2 and
 * 96 zero bytes (its verdict is 0 and it moves no latest message anyway).  Both asynchronous on `stream`; bits_stride <= 256. */
int b2_votes_group_dev(b2_ctx* ctx, const uint32_t* d_vote, const uint32_t* d_vote_off, uint32_t n_votes, const uint32_t* d_members, const uint32_t* d_off,
                       uint32_t n_committees, uint64_t n_sig, uint32_t bits_stride, const uint8_t* d_sig96, uint32_t c_begin, uint32_t c_end,
                       uint8_t* d_sig96_out, uint32_t* d_members_out, uint32_t* d_pos_out, uint32_t* d_seg_off, uint32_t* d_seg_off_loc,
                       uint8_t* d_bits_out, uint8_t* d_agg_bits_out, void* stream);
int b2_votes_empty_dev(b2_ctx* ctx, const uint8_t* d_bits, uint32_t bits_stride, uint32_t n_votes, uint8_t* d_agg_sig96, int32_t* d_agg_status,
                       void* stream);
/* ---- attestation intake: one epoch of unaggregated Attestations straight off the wire (pos-evolution.md:714-717; each with one member's
 * AttestationData, one set bit and one signature) checked and turned into the vote form's inputs above.  Target epoch e, committee c of
 * the epoch = (data.slot - start_slot(e)) * committees_per_slot + data.index with members d_off[c] .. d_off[c+1] (the layout of the
 * epoch's b2_votes_group_dev call; n_committees = slots_per_epoch * committees_per_slot).  wire / woff are the encodings of
 * b2_attestations_decode, wire_len the wire's length in bytes.  Every attestation gets exactly one status, the first failing check:
 *    0  kept
 *    1  malformed container; also a woff row that is reversed or ends past wire_len
 *    2  empty Bitlist or no delimiter
 *    3  more bits than 8 * bits_stride
 *    4  not exactly one bit set
 *    5  Bitlist length != the size of its committee (:730); a malformed committee row (device form) matches no length
 *    6  data.slot outside epoch e, or data.index >= committees_per_slot (:725-727)
 *    7  data.target.epoch != e
 *    8  current_slot < data.slot + 1
 *    9  beacon_block_root is not a block of the device tree
 *   10  target.root is not a block of the device tree
 *   11  slot(beacon_block_root) > data.slot
 *   12  target.root != get_ancestor(beacon_block_root, start_slot(e)); a walk that reaches the tree's root while still above
 *       start_slot(e) is not the ancestor
 *   13  duplicate: an earlier attestation in list order that passed checks 1-12 holds the same (committee, position)
 * Checks 9-12 are validate_on_attestation's (upstream fork-choice spec v1.2.0, :963-979) with store.blocks = the tree on the device:
 * the blocks since the last b2_tree_prune, with the slots given to b2_tree_load / b2_tree_add.  Checks 5-8 are process_attestation's
 * (:724-730); validate_target_epoch_against_current_time is made for the whole batch: an epoch e that is neither current_slot's epoch nor
 * the one before it is B2_EINVAL.  Outputs, the arrays the vote form takes:
 *   vote u32[n_sig]           vote[d_off[c] + p] = the vote id of the attestation kept at position p, or 0xFFFFFFFF.  A committee's kept
 *                             attestations are grouped by their 128 data bytes (SSZ serialisation is injective); its vote ids are in the
 *                             order of each group's smallest position.  A committee with nothing kept has one placeholder id.
 *   vote_off u32[n_committees + 1]   written on the device;
 *   sig96 u8[n_sig][96]       the kept signatures in committee order, zero where nothing is kept;
 *   per vote v < max_votes    data128 u8[128], msg32 = compute_signing_root(data, domain32), source and target epoch (u64), block_idx =
 *                             the tree id of beacon_block_root; a placeholder has zero data and message and block 0.
 * An epoch with more than max_votes votes keeps its true counts in vote_off; only the first max_votes rows are written.  domain32 =
 * get_domain(DOMAIN_BEACON_ATTESTER, e), a host pointer read when the call is made.
 * b2_attestation_intake_dev is asynchronous on `stream` and self-guarding: a woff row that is reversed or ends past wire_len is status 1,
 * a committee row that is reversed, ends past n_sig or exceeds 8 * bits_stride gets only its placeholder and its positions are not written
 * (both B2_GUARD_BAD_ROW); nothing is read or written out of bounds.  The intakes of one context run one after another (they share its
 * scratch), and the tree must not change while one is in flight.  b2_attestation_intake takes host arrays and returns when done; it
 * checks woff (starts at 0, never decreases, ends inside the wire) and d_off (the same, no committee larger than 8 * bits_stride) first,
 * and a rejected call (B2_EINVAL: these, a committee count that does not match, no loaded tree, a bad epoch, bits_stride == 0 or > 256,
 * n_att or max_votes == 0) writes no output and changes nothing; rows past the epoch's vote count are zero. */
int b2_attestation_intake_dev(b2_ctx* ctx, const uint8_t* d_wire, uint64_t wire_len, const uint32_t* d_woff, uint32_t n_att, const uint32_t* d_off,
                              uint32_t n_committees, uint64_t n_sig, uint32_t committees_per_slot, uint32_t slots_per_epoch, uint32_t bits_stride,
                              uint64_t epoch, uint64_t current_slot, const uint8_t* domain32, uint32_t max_votes, int32_t* d_status_out,
                              uint32_t* d_vote_out, uint32_t* d_vote_off_out, uint8_t* d_sig96_out, uint8_t* d_data128_out, uint8_t* d_msg32_out,
                              uint64_t* d_source_epoch_out, uint64_t* d_target_epoch_out, uint32_t* d_block_idx_out, void* stream);
int b2_attestation_intake(b2_ctx* ctx, const uint8_t* wire, uint64_t wire_len, const uint32_t* woff, uint32_t n_att, const uint32_t* off,
                          uint32_t n_committees, uint32_t committees_per_slot, uint32_t slots_per_epoch, uint32_t bits_stride, uint64_t epoch,
                          uint64_t current_slot, const uint8_t* domain32, uint32_t max_votes, int32_t* status_out, uint32_t* vote_out,
                          uint32_t* vote_off_out, uint8_t* sig96_out, uint8_t* data128_out, uint8_t* msg32_out, uint64_t* source_epoch_out,
                          uint64_t* target_epoch_out, uint32_t* block_idx_out);
/* ---- SingleAttestation intake: one epoch of Electra's unaggregated attestations (EIP-7549; the beacon_attestation_{subnet_id} topic of
 * the upstream Electra p2p spec) checked and turned into the same vote form's inputs as b2_attestation_intake.  Container:
 *   SingleAttestation{committee_index u64, attester_index u64, data AttestationData, signature BLSSignature}: 240 fixed bytes
 * wire / woff = the encodings back to back and their byte offsets, wire_len the wire's bytes.  subnet[a] = the subnet id of the topic item
 * a arrived on, subnet_count = ATTESTATION_SUBNET_COUNT.  Committee c of the epoch = (data.slot - start_slot(e)) * committees_per_slot +
 * committee_index, members d_members[d_off[c] .. d_off[c+1]) (the layout of b2_attestation_intake; precondition: the committees are
 * pairwise disjoint, as get_beacon_committee makes them).  Every item gets exactly one status, the first failing check:
 *    0  kept
 *    1  the item is not 240 bytes; also a woff row that is reversed or ends past wire_len
 *    2  data.index != 0
 *    3  committee_index >= committees_per_slot
 *    4  data.slot outside epoch e
 *    5  compute_subnet_for_attestation(committees_per_slot, data.slot, committee_index) != subnet[a]
 *    6  data.target.epoch != e
 *    7  current_slot < data.slot + 1
 *    8  attester_index is not a member of committee (data.slot, committee_index); a malformed committee row (device form) has no members
 *    9-12  b2_attestation_intake's 9-12 (the same tree walk)
 *   13  duplicate: an earlier item in list order that passed checks 1-12 has the same attester_index (the same committee position)
 * The attester's position is the smallest one of the committee that holds attester_index.  Signatures are not checked per item: the
 * epoch pipeline verifies each vote's aggregate.  Outputs, max_votes, domain32, the device form's guards and the order of the calls
 * sharing scratch are b2_attestation_intake's; data128 and msg32 are those of the data as signed (data.index == 0).  The host form
 * refuses (B2_EINVAL, nothing written) what b2_attestation_intake refuses, and a missing subnet or members array or subnet_count == 0;
 * both forms refuse n_att == 0, so every call they accept has items and needs its subnet array. */
int b2_single_attestation_intake_dev(b2_ctx* ctx, const uint8_t* d_wire, uint64_t wire_len, const uint32_t* d_woff, uint32_t n_att,
                                     const uint32_t* d_subnet, uint32_t subnet_count, const uint32_t* d_members, const uint32_t* d_off,
                                     uint32_t n_committees, uint64_t n_sig, uint32_t committees_per_slot, uint32_t slots_per_epoch, uint32_t bits_stride,
                                     uint64_t epoch, uint64_t current_slot, const uint8_t* domain32, uint32_t max_votes, int32_t* d_status_out,
                                     uint32_t* d_vote_out, uint32_t* d_vote_off_out, uint8_t* d_sig96_out, uint8_t* d_data128_out, uint8_t* d_msg32_out,
                                     uint64_t* d_source_epoch_out, uint64_t* d_target_epoch_out, uint32_t* d_block_idx_out, void* stream);
int b2_single_attestation_intake(b2_ctx* ctx, const uint8_t* wire, uint64_t wire_len, const uint32_t* woff, uint32_t n_att, const uint32_t* subnet,
                                 uint32_t subnet_count, const uint32_t* members, const uint32_t* off, uint32_t n_committees, uint32_t committees_per_slot,
                                 uint32_t slots_per_epoch, uint32_t bits_stride, uint64_t epoch, uint64_t current_slot, const uint8_t* domain32,
                                 uint32_t max_votes, int32_t* status_out, uint32_t* vote_out, uint32_t* vote_off_out, uint8_t* sig96_out,
                                 uint8_t* data128_out, uint8_t* msg32_out, uint64_t* source_epoch_out, uint64_t* target_epoch_out,
                                 uint32_t* block_idx_out);
/* ---- aggregated-attestation intake: one target epoch e of SignedAggregateAndProof messages from gossip (the beacon_aggregate_and_proof
 * topic of the upstream phase 0 p2p spec), checked and verified on the device.  Containers (upstream phase 0):
 *   AggregateAndProof{aggregator_index u64, aggregate Attestation, selection_proof BLSSignature}
 *   SignedAggregateAndProof{message AggregateAndProof, signature BLSSignature}
 * wire / woff = the SSZ encodings back to back and their byte offsets (as b2_attestations_decode takes them), wire_len the wire's bytes.
 * Committee c of the epoch = (data.slot - start_slot(e)) * committees_per_slot + data.index, members d_members[d_off[c] .. d_off[c+1])
 * (the layout of b2_attestation_intake; precondition: the committees are pairwise disjoint, as get_beacon_committee makes them).
 * domains96 (host pointer) = get_domain(., D, e) for D = DOMAIN_BEACON_ATTESTER, DOMAIN_SELECTION_PROOF, DOMAIN_AGGREGATE_AND_PROOF, back to
 * back.  target_aggregators = TARGET_AGGREGATORS_PER_COMMITTEE, propagation_slot_range = ATTESTATION_PROPAGATION_SLOT_RANGE.
 * Every item gets exactly one status, the first failing check in this order (the class is what gossip scoring reads):
 *    0  accept
 *    1  reject  malformed outer, inner or nested container (offsets, lengths, trailing bytes); also a woff row that is reversed or ends
 *               past wire_len
 *    2  reject  empty Bitlist or no delimiter
 *    3  reject  more bits than 8 * bits_stride
 *    4  reject  data.index >= committees_per_slot
 *    5  ignore  not data.slot <= current_slot <= data.slot + propagation_slot_range
 *    6  reject  data.target.epoch != compute_epoch_at_slot(data.slot)
 *    7  (other) compute_epoch_at_slot(data.slot) != e: the item belongs to the other epoch's call
 *    8  reject  Bitlist length != committee size; a malformed committee row (device form) matches no length
 *    9  reject  no bit set
 *   10  ignore  an earlier ACCEPTED item of the call has byte-equal AttestationData and bits that cover this item's
 *   11  ignore  an earlier ACCEPTED item of the call has the same aggregator_index
 *   12  reject  is_aggregator is false: bytes_to_uint64(hash(selection_proof)[0:8]) % max(1, len(committee) // target_aggregators) != 0
 *   13  reject  aggregator_index is not in the committee
 *   14  reject  the selection proof fails Verify(pubkey(aggregator), compute_signing_root(data.slot, selection domain))
 *   15  reject  the signature fails Verify(pubkey(aggregator), compute_signing_root(AggregateAndProof, aggregate_and_proof domain))
 *   16  reject  the aggregate fails FastAggregateVerify over the selected members and the attestation signing root
 *   17  ignore  beacon_block_root is not a block of the device tree
 *   18  reject  target.root is not a block of the device tree
 *   19  reject  slot(beacon_block_root) > data.slot
 *   20  reject  target.root != get_ancestor(beacon_block_root, start_slot(e))
 * 17-20 are b2_attestation_intake's 9-12 (the same tree walk).  Checks 10 and 11 read only earlier items of the same call that end with
 * status 0: each item gets the status it would get if the items arrived one by one in list order at a node whose seen-caches were empty
 * when the call began (the caller keeps the caches across calls).  e must be current_slot's epoch or the one before it.
 * Outputs per item (n items; zero rows, 0xFFFFFFFF ids for an item that did not decode, statuses 1-3):
 *   committee u32        c, or 0xFFFFFFFF for statuses 1-7
 *   data_id u32          the smallest list index with byte-equal AttestationData
 *   bits u8[bits_stride] the aggregation bits, delimiter removed, zero padded
 *   sig96, msg32         the aggregate signature as on the wire; compute_signing_root(data, attester domain)
 *   target_epoch u64, block_idx u32   data.target.epoch; the tree id of beacon_block_root (0xFFFFFFFF when absent)
 *   members u32[n][8 * bits_stride], item_off u32[n+1]   item a's member row = its committee, zero padded, and item_off[a] = 8 * bits_stride * a:
 *                        with bits and accept = (status == 0) these are what b2_latest_messages_update_dev (on_attestation of the accepted
 *                        aggregates) and b2_fast_aggregate_verify_dev take, and the rows the FastAggregateVerify of check 16 consumed.
 * b2_aggregate_and_proof_intake_dev is asynchronous on `stream` and self-guarding: a woff row that is reversed or ends past wire_len is
 * status 1 and a committee row that is reversed, ends past n_sig (the members' length) or exceeds 8 * bits_stride is status 8 (both
 * B2_GUARD_BAD_ROW); an aggregator index that is not a member never reaches the registry (status 13), and a member index >= n_validators
 * fails the checks that read it (B2_GUARD_BAD_INDEX); nothing is read or written out of bounds.  It shares scratch with the intake (the
 * two run one after another) and with the synchronous verify entry points: the verify buffers of pipeline slot 0 (b2_fast_aggregate_verify,
 * _pks, _dev, b2_epoch_dev) and the AggregateVerify buffers (b2_aggregate_verify, _pks, _dev); enqueue those on the same stream.  The
 * tree and the registry must not change while a call is in flight.  b2_aggregate_and_proof_intake takes host arrays and returns when
 * done; it checks woff (starts at 0, never decreases, ends inside the wire) and off (the same, no committee larger than 8 * bits_stride)
 * first, and a rejected call (B2_EINVAL: these, a committee count other than slots_per_epoch * committees_per_slot, no registry or tree,
 * a bad epoch, bits_stride == 0 or > 256, target_aggregators == 0, n == 0) writes no output and changes nothing. */
int b2_aggregate_and_proof_intake_dev(b2_ctx* ctx, const uint8_t* d_wire, uint64_t wire_len, const uint32_t* d_woff, uint32_t n, const uint32_t* d_members,
                                      const uint32_t* d_off, uint32_t n_committees, uint64_t n_sig, uint32_t committees_per_slot, uint32_t slots_per_epoch,
                                      uint32_t bits_stride, uint64_t epoch, uint64_t current_slot, const uint8_t* domains96, uint32_t target_aggregators,
                                      uint64_t propagation_slot_range, int32_t* d_status_out, uint32_t* d_committee_out, uint32_t* d_data_id_out,
                                      uint8_t* d_bits_out, uint8_t* d_sig96_out, uint8_t* d_msg32_out, uint64_t* d_target_epoch_out,
                                      uint32_t* d_block_idx_out, uint32_t* d_members_out, uint32_t* d_item_off_out, void* stream);
int b2_aggregate_and_proof_intake(b2_ctx* ctx, const uint8_t* wire, uint64_t wire_len, const uint32_t* woff, uint32_t n, const uint32_t* members,
                                  const uint32_t* off, uint32_t n_committees, uint32_t committees_per_slot, uint32_t slots_per_epoch, uint32_t bits_stride,
                                  uint64_t epoch, uint64_t current_slot, const uint8_t* domains96, uint32_t target_aggregators,
                                  uint64_t propagation_slot_range, int32_t* status_out, uint32_t* committee_out, uint32_t* data_id_out, uint8_t* bits_out,
                                  uint8_t* sig96_out, uint8_t* msg32_out, uint64_t* target_epoch_out, uint32_t* block_idx_out, uint32_t* members_out,
                                  uint32_t* item_off_out);
/* ---- process_attestation (pos-evolution.md:722-754) for the attestations of a run of blocks of one chain in one epoch e, block-atomic as
 * on_block's state_transition (:1008-1009).  Inputs:
 *   wire, woff[n_att+1], wire_len   the attestations' SSZ encodings back to back (b2_attestations_decode's form), in block order and list
 *                                   order within a block
 *   block_off[n_blocks+1]           block b holds attestations [block_off[b], block_off[b+1])
 *   block_slot[n_blocks]            the state.slot of each block: strictly increasing, all in epoch e = block_slot[0] / slots_per_epoch
 *   members, off[n_committees+1]    the committees of e - 1 (cps_prev * slots_per_epoch rows), then those of e (cps_cur * slots_per_epoch
 *                                   rows; n_committees = their sum): committee (E, slot, index) = (E == e ? cps_prev * slots_per_epoch : 0) + (slot - start(E)) *
 *                                   cps_E + index.  At e = 0 there is no previous epoch and cps_prev is 0.
 *   chain_roots u8[2 * slots_per_epoch][32]   the root of slot s at s + slots_per_epoch - start(e), state.block_roots[s %
 *                                   SLOTS_PER_HISTORICAL_ROOT] as this chain sees it; only slots below the including block's slot are read
 *   justified80 (host)              previous_justified_checkpoint, then current_justified_checkpoint, 40 SSZ bytes each (epoch u64 LE || root)
 *   domains64 (host)                get_domain(DOMAIN_BEACON_ATTESTER, e - 1), then the same for e
 * plus MIN_ATTESTATION_INCLUSION_DELAY (> 0), bits_stride (1..256), EFFECTIVE_BALANCE_INCREMENT and get_base_reward_per_increment;
 * integer_squareroot(slots_per_epoch) is computed inside.  Each attestation gets the first check it fails, in process_attestation's order:
 *    0  passes every check
 *    1  malformed container, or a woff row that is reversed or ends past wire_len, or an attestation in no block's row
 *    2  empty Bitlist or no delimiter                  3  more bits than 8 * bits_stride
 *    4  target.epoch is neither e - 1 nor e (:724)     5  target.epoch != compute_epoch_at_slot(data.slot) (:725)
 *    6  not data.slot + MIN_ATTESTATION_INCLUSION_DELAY <= block slot <= data.slot + SLOTS_PER_EPOCH (:726)
 *    7  data.index >= committees_per_slot of the target epoch (:727)
 *    8  Bitlist length != committee size (:730); a malformed committee row matches no length
 *    9  data.source != the justified checkpoint of the target epoch (:733, is_matching_source)
 *   10  no bit set (:736, is_valid_indexed_attestation on empty indices)     11  FastAggregateVerify fails (:736)
 * Outputs per attestation: status; flag_mask (bit f = participation flag f, get_attestation_participation_flag_indices with inclusion_delay =
 * block slot - data.slot; 0 unless checks 1-9 pass); numerator u64 (proposer_reward_numerator of :745-749, 0 where not applied).  Per block:
 * block_status (0 applied, 1 invalid: its row is malformed or it holds a nonzero status, 2 valid but after the first invalid block);
 * block_first, the list index of its first failing attestation or 0xFFFFFFFF; block_reward, the sum over its attestations of numerator //
 * 448 (:752-754, the proposer's increase_balance).  n_applied: the blocks applied, those before the first invalid one.  They set the flags of
 * the attestations with target e in participation table 0 and of those with target e - 1 in table 1, order-exact over (block, list) order
 * (a repeated attestation is valid and earns nothing); rewards read the registry's effective balances; nothing of the first invalid block
 * or of a later one changes a table.  b2_set_verify_mode applies to the FastAggregateVerify.
 * b2_block_attestations_dev is asynchronous on `stream` and self-guarding: a woff row that is reversed or ends past wire_len is status 1, a
 * committee row that is reversed, ends past n_sig or exceeds 8 * bits_stride is status 8, and a block whose block_off row is reversed or
 * ends past n_att, whose slot is outside e or not above the previous block's, is invalid (all B2_GUARD_BAD_ROW); a member index >=
 * n_validators fails FastAggregateVerify (B2_GUARD_BAD_INDEX); nothing is read or written out of bounds.  It shares the verify buffers of
 * pipeline slot 0 with the synchronous verify entry points and the aggregate intake: enqueue those on the same stream.  The registry and
 * the participation tables must not change while a call is in flight.  b2_block_attestations takes host arrays and returns when done; a
 * rejected call (B2_EINVAL: no registry or a participation table not loaded, a woff, block_off or off row that does not start at 0 or
 * decreases, woff ending past the wire, block_off not ending at n_att, a committee larger than 8 * bits_stride, block slots that do not
 * increase strictly or leave one epoch, cps_prev != 0 exactly when e == 0, a committee count other than slots_per_epoch * (cps_prev +
 * cps_cur) (the device form refuses that too), bits_stride 0 or > 256, n_att == 0 or n_blocks == 0) writes no
 * output and changes nothing. */
int b2_block_attestations_dev(b2_ctx* ctx, const uint8_t* d_wire, uint64_t wire_len, const uint32_t* d_woff, uint32_t n_att, const uint32_t* d_block_off,
                              const uint64_t* d_block_slot, uint32_t n_blocks, const uint32_t* d_members, const uint32_t* d_off, uint32_t n_committees,
                              uint64_t n_sig,
                              uint32_t cps_prev, uint32_t cps_cur, const uint8_t* d_chain_roots, const uint8_t* justified80, const uint8_t* domains64,
                              uint32_t slots_per_epoch, uint32_t min_inclusion_delay, uint32_t bits_stride, uint64_t effective_balance_increment,
                              uint64_t base_reward_per_increment, int32_t* d_status_out, uint8_t* d_flag_mask_out, uint64_t* d_numerator_out,
                              int32_t* d_block_status_out, uint32_t* d_block_first_out, uint64_t* d_block_reward_out, uint32_t* d_n_applied_out,
                              void* stream);
int b2_block_attestations(b2_ctx* ctx, const uint8_t* wire, uint64_t wire_len, const uint32_t* woff, uint32_t n_att, const uint32_t* block_off,
                          const uint64_t* block_slot, uint32_t n_blocks, const uint32_t* members, const uint32_t* off, uint32_t n_committees,
                          uint32_t cps_prev, uint32_t cps_cur, const uint8_t* chain_roots, const uint8_t* justified80, const uint8_t* domains64, uint32_t slots_per_epoch,
                          uint32_t min_inclusion_delay, uint32_t bits_stride, uint64_t effective_balance_increment, uint64_t base_reward_per_increment,
                          int32_t* status_out, uint8_t* flag_mask_out, uint64_t* numerator_out, int32_t* block_status_out, uint32_t* block_first_out,
                          uint64_t* block_reward_out, uint32_t* n_applied_out);
/* ---- process_attestation for the Electra (EIP-7549) on-chain Attestation, with Deneb's (EIP-7045) inclusion window and flags (upstream
 * consensus-specs, Deneb and Electra beacon-chain.md), for the attestations of a run of blocks of one chain in one epoch e.  The inputs and
 * outputs are b2_block_attestations', except:
 *   wire                            Electra encodings: offset u32 | AttestationData 128 | signature 96 | committee_bits ceil(M / 8) |
 *                                   aggregation_bits Bitlist[max_validators_per_committee * M], M = max_committees_per_slot (1..64)
 *   max_validators_per_committee    with M, the Bitlist's limit (their product < 2^31)
 *   row_max (device form only)      the largest member count of one slot's committees over e - 1 and e (> 0); the host form computes it
 * An attestation names the committees (data.slot, i) of the bits i set in committee_bits, and its Bitlist is their bit rows back to back in
 * increasing i.  Each attestation gets the first check it fails:
 *    0  passes every check
 *    1  malformed container (truncated, offset != fixed size, a committee_bits padding bit set), a woff row that is reversed or ends past
 *       wire_len, or an attestation in no block's row
 *    2  empty Bitlist or no delimiter                  3  more bits than max_validators_per_committee * M
 *    4  target.epoch is neither e - 1 nor e            5  target.epoch != compute_epoch_at_slot(data.slot)
 *    6  data.slot + MIN_ATTESTATION_INCLUSION_DELAY > block slot (no upper bound since Deneb)
 *    7  data.index != 0
 *    8-10  the committees by increasing index: 8 an index >= committees_per_slot of the target epoch; 10 its bit row runs past the Bitlist's
 *       end; 9 no bit of its row set.  After them, 10 when the Bitlist's length is not their total size.
 *   11  data.source != the justified checkpoint of the target epoch
 *   12  no committee bit set (is_valid_indexed_attestation on empty indices)          13  FastAggregateVerify fails
 * flag_mask is 0 unless checks 1-11 pass; its flags are Deneb's: timely source at inclusion delay <= integer_squareroot(slots_per_epoch),
 * timely target whenever the target root matches, timely head when the target and head roots match at delay MIN_ATTESTATION_INCLUSION_DELAY.
 * numerator, block_status, block_first, block_reward, n_applied, the two participation tables, block atomicity and b2_set_verify_mode are as
 * in b2_block_attestations.  Committees are disjoint.
 * b2_block_attestations_electra_dev is asynchronous on `stream` and self-guarding as b2_block_attestations_dev is; a committee row that is
 * reversed or ends past n_sig, or whose committees add up to more than row_max members, is status 10 (B2_GUARD_BAD_ROW).  It shares pipeline
 * slot 0's verify buffers as that call does.  b2_block_attestations_electra takes host arrays and returns when done; a rejected call (B2_EINVAL:
 * b2_block_attestations' refusals without those on bits_stride, and M outside 1..64, max_validators_per_committee 0 or its product with M
 * >= 2^31, n_att times the padded row >= 2^32 members) writes no output and changes nothing. */
int b2_block_attestations_electra_dev(b2_ctx* ctx, const uint8_t* d_wire, uint64_t wire_len, const uint32_t* d_woff, uint32_t n_att,
                                      const uint32_t* d_block_off, const uint64_t* d_block_slot, uint32_t n_blocks, const uint32_t* d_members,
                                      const uint32_t* d_off, uint32_t n_committees, uint64_t n_sig, uint32_t cps_prev, uint32_t cps_cur,
                                      const uint8_t* d_chain_roots, const uint8_t* justified80, const uint8_t* domains64, uint32_t slots_per_epoch,
                                      uint32_t min_inclusion_delay, uint32_t max_committees_per_slot, uint32_t max_validators_per_committee,
                                      uint32_t row_max, uint64_t effective_balance_increment, uint64_t base_reward_per_increment,
                                      int32_t* d_status_out, uint8_t* d_flag_mask_out, uint64_t* d_numerator_out, int32_t* d_block_status_out,
                                      uint32_t* d_block_first_out, uint64_t* d_block_reward_out, uint32_t* d_n_applied_out, void* stream);
int b2_block_attestations_electra(b2_ctx* ctx, const uint8_t* wire, uint64_t wire_len, const uint32_t* woff, uint32_t n_att, const uint32_t* block_off,
                                  const uint64_t* block_slot, uint32_t n_blocks, const uint32_t* members, const uint32_t* off, uint32_t n_committees,
                                  uint32_t cps_prev, uint32_t cps_cur, const uint8_t* chain_roots, const uint8_t* justified80, const uint8_t* domains64,
                                  uint32_t slots_per_epoch, uint32_t min_inclusion_delay, uint32_t max_committees_per_slot,
                                  uint32_t max_validators_per_committee, uint64_t effective_balance_increment, uint64_t base_reward_per_increment,
                                  int32_t* status_out, uint8_t* flag_mask_out, uint64_t* numerator_out, int32_t* block_status_out,
                                  uint32_t* block_first_out, uint64_t* block_reward_out, uint32_t* n_applied_out);
/* ---- One slot of sync committee messages from gossip: SyncCommitteeMessage (pos-evolution.md:548-557) checked as the sync_committee_{subnet_id}
 * topics of the upstream Altair p2p spec require, grouped by beacon_block_root, and summed into each subnet's SyncCommitteeContribution and each
 * root's SyncAggregate as process_sync_committee_contributions of the upstream Altair validator spec builds them.  Inputs:
 *   wire, woff[n+1], wire_len     the messages' SSZ encodings back to back: slot u64 | beacon_block_root 32 | validator_index u64 | signature 96
 *   subnet[n]                     the subnet id of the topic each message arrived on
 *   position_validator[committee_size]   the registry index of each position of the sync committee (the first registry index of its key, as
 *                                 process_sync_aggregate maps it); a validator may hold several positions
 *   committee_size, subnet_count  subcommittee size = committee_size / subnet_count; subnet s holds positions [s * size / count, (s + 1) * ...)
 *   current_slot, domain32 (host) get_domain(state, DOMAIN_SYNC_COMMITTEE, epoch of current_slot)
 * Each message gets the first check it fails (IGNORE or REJECT as the p2p spec classes it):
 *    0  accepted
 *    1  REJECT  not 144 bytes, or a woff row that is reversed or ends past wire_len
 *    2  IGNORE  slot != current_slot (clock disparity is the caller's)
 *    3  REJECT  validator_index >= n_validators
 *    4  REJECT  subnet_id is not one of the validator's subnets (no position p of it with p / subcommittee size == subnet_id), subnet_id >= count
 *    5  IGNORE  an earlier message of the list with the same (validator_index, subnet_id) was accepted (checked before the signature)
 *    6  REJECT  Verify(registry key, sha256(beacon_block_root || domain32), signature) fails, a key that failed KeyValidate included
 * Outputs: status i32[n]; root_id u32[n], the accepted messages' distinct roots numbered by first occurrence in the list, 0xFFFFFFFF for the
 * others; roots32 u8[n][32] and n_roots u32[1] (rows >= n_roots are zero).  Per (root r, subnet s), row r * subnet_count + s:
 * contrib_bits u8[n * subnet_count][ceil(subcommittee size / 8)], a Bitvector with bit i set iff the validator at position s * subcommittee size
 * + i has an accepted message on subnet s naming root r; contrib_sig96 the sum of those validators' signatures, one term per set bit (a
 * validator at k positions of the subnet counts k times, as eth_fast_aggregate_verify over the positions needs); contrib_present u8, 0 where no
 * bit is set (bits and signature then zero).  Per root: agg_bits u8[n][ceil(committee_size / 8)], the subnets' rows concatenated bit by bit,
 * and agg_sig96, the sum over every set position (bls.Aggregate of the present contributions): the SyncAggregate a proposer includes for that
 * root, which b2_sync_aggregate_verify accepts.  Rows of roots >= n_roots are zero.
 * b2_sync_committee_messages_dev is asynchronous on `stream` and self-guarding: a reversed woff row or one past wire_len is status 1
 * (B2_GUARD_BAD_ROW), a bad subnet is status 4, and a position_validator entry >= n_validators matches nothing (B2_GUARD_BAD_INDEX).  It needs
 * the registry (not b2_sync_committee_load's tables) and shares the AggregateVerify buffers with b2_aggregate_verify[_pks, _dev] and the
 * intakes: enqueue those and this call on one stream.  The registry must not change while a call is in flight.
 * b2_sync_committee_messages takes host arrays and returns when done; a rejected call (B2_EINVAL: a woff that does not start at 0, decreases or
 * ends past the wire, a position_validator entry >= n_validators, committee_size not a multiple of subnet_count or above 1024, no registry,
 * n == 0) writes no output and changes nothing. */
int b2_sync_committee_messages_dev(b2_ctx* ctx, const uint8_t* d_wire, uint64_t wire_len, const uint32_t* d_woff, uint32_t n, const uint32_t* d_subnet,
                                   const uint32_t* d_position_validator, uint32_t committee_size, uint32_t subnet_count, uint64_t current_slot,
                                   const uint8_t* domain32, int32_t* d_status_out, uint32_t* d_root_id_out, uint8_t* d_roots32_out,
                                   uint32_t* d_n_roots_out, uint8_t* d_contrib_bits_out, uint8_t* d_contrib_sig96_out, uint8_t* d_contrib_present_out,
                                   uint8_t* d_agg_bits_out, uint8_t* d_agg_sig96_out, void* stream);
int b2_sync_committee_messages(b2_ctx* ctx, const uint8_t* wire, uint64_t wire_len, const uint32_t* woff, uint32_t n, const uint32_t* subnet,
                               const uint32_t* position_validator, uint32_t committee_size, uint32_t subnet_count, uint64_t current_slot,
                               const uint8_t* domain32, int32_t* status_out, uint32_t* root_id_out, uint8_t* roots32_out, uint32_t* n_roots_out,
                               uint8_t* contrib_bits_out, uint8_t* contrib_sig96_out, uint8_t* contrib_present_out, uint8_t* agg_bits_out,
                               uint8_t* agg_sig96_out);
/* ---- One slot of sync committee contributions from gossip: SignedContributionAndProof checked as the sync_committee_contribution_and_proof
 * topic of the upstream Altair p2p spec requires, and per beacon_block_root the SyncAggregate process_sync_committee_contributions (upstream
 * Altair validator spec) builds from the best accepted contribution of each subnet.  Inputs:
 *   wire, woff[n+1], wire_len     the items' SSZ encodings back to back, 344 + ceil(sub / 8) bytes each (every field is fixed-size):
 *                                 ContributionAndProof (aggregator_index u64 | SyncCommitteeContribution (slot u64 | beacon_block_root 32 |
 *                                 subcommittee_index u64 | aggregation_bits Bitvector[sub] | signature 96) | selection_proof 96) | signature 96
 *   position_validator[committee_size]   the registry index of each position of the sync committee, as for b2_sync_committee_messages
 *   committee_size, subnet_count  sub = committee_size / subnet_count; subnet s holds positions [s * sub, (s + 1) * sub)
 *   current_slot
 *   domains96 (host)              get_domain of current_slot's epoch for DOMAIN_SYNC_COMMITTEE, DOMAIN_SYNC_COMMITTEE_SELECTION_PROOF and
 *                                 DOMAIN_CONTRIBUTION_AND_PROOF, back to back
 *   target_aggregators            TARGET_AGGREGATORS_PER_SYNC_SUBCOMMITTEE (> 0)
 * Each item gets the first check it fails (IGNORE or REJECT as the p2p spec classes it):
 *    0  accepted
 *    1  REJECT  not 344 + ceil(sub / 8) bytes, a Bitvector bit at or past sub set, or a woff row that is reversed or ends past wire_len
 *    2  IGNORE  contribution.slot != current_slot (clock disparity is the caller's)
 *    3  REJECT  subcommittee_index >= subnet_count
 *    4  REJECT  no aggregation bit set
 *    5  REJECT  is_sync_committee_aggregator is false: bytes_to_uint64(hash(selection_proof)[0:8]) % max(1, sub // target_aggregators) != 0
 *    6  REJECT  aggregator_index >= n_validators
 *    7  REJECT  aggregator_index holds no position of subnet subcommittee_index (registry indices compared)
 *    8  IGNORE  an earlier ACCEPTED item has the same (beacon_block_root, subcommittee_index) and bits that include this item's
 *    9  IGNORE  an earlier ACCEPTED item has the same (aggregator_index, subcommittee_index), on any root
 *   10  REJECT  the selection proof fails Verify(key(aggregator), compute_signing_root(SyncAggregatorSelectionData(slot, subcommittee_index),
 *               selection domain))
 *   11  REJECT  the signature fails Verify(key(aggregator), compute_signing_root(ContributionAndProof, contribution_and_proof domain))
 *   12  REJECT  the contribution's signature fails FastAggregateVerify over the registry keys of the set positions of its subnet (a validator
 *               at k positions counts k times) and compute_signing_root(beacon_block_root, sync committee domain)
 * A key that failed KeyValidate fails 10, 11 or 12.  Checks 8 and 9 read only earlier items of the same call that end with status 0: each
 * item gets the status it would get if the items arrived one by one in list order at a node whose seen-caches were empty when the call
 * began (the caller keeps the caches across calls).
 * Outputs (n items): status i32[n]; root_id u32[n], the accepted items' distinct roots numbered by first accepted occurrence, 0xFFFFFFFF for
 * the others; roots32 u8[n][32] and n_roots u32[1] (rows >= n_roots are zero); best u32[n][subnet_count], per (root, subnet) the list index
 * of the accepted item with the most set bits (ties to the smaller index), 0xFFFFFFFF where there is none; agg_bits u8[n][ceil(committee_size
 * / 8)] and agg_sig96 u8[n][96], per root the SyncAggregate of its best contributions (bit s * sub + i = bit i of best[r][s]'s row, signature
 * bls.Aggregate of their signatures): what a proposer includes, and what b2_sync_aggregate_verify accepts.  Rows of roots >= n_roots are
 * zero, except best's, which are 0xFFFFFFFF (no item).  The accepted contributions themselves are the caller's wire bytes.
 * b2_sync_contribution_and_proof_intake_dev is asynchronous on `stream` and self-guarding: a reversed woff row or one past wire_len is status
 * 1 (B2_GUARD_BAD_ROW), and a position_validator entry >= n_validators matches nothing (B2_GUARD_BAD_INDEX); nothing is read or written out
 * of bounds.  It needs the registry (not b2_sync_committee_load's tables) and shares the AggregateVerify buffers and the verify buffers of
 * pipeline slot 0 with b2_aggregate_verify[_pks, _dev], b2_fast_aggregate_verify[_pks, _dev], b2_epoch_dev and the intakes: enqueue those and
 * this call on one stream.  b2_set_verify_mode applies to its FastAggregateVerify.  The registry must not change while a call is in flight.
 * b2_sync_contribution_and_proof_intake takes host arrays and returns when done; a rejected call (B2_EINVAL: a woff that does not start at 0,
 * decreases or ends past the wire, a position_validator entry >= n_validators, committee_size not a multiple of subnet_count or above 1024,
 * target_aggregators == 0, no registry, n == 0 or n >= 2^24) writes no output and changes nothing. */
int b2_sync_contribution_and_proof_intake_dev(b2_ctx* ctx, const uint8_t* d_wire, uint64_t wire_len, const uint32_t* d_woff, uint32_t n,
                                              const uint32_t* d_position_validator, uint32_t committee_size, uint32_t subnet_count,
                                              uint64_t current_slot, const uint8_t* domains96, uint32_t target_aggregators, int32_t* d_status_out,
                                              uint32_t* d_root_id_out, uint8_t* d_roots32_out, uint32_t* d_n_roots_out, uint32_t* d_best_out,
                                              uint8_t* d_agg_bits_out, uint8_t* d_agg_sig96_out, void* stream);
int b2_sync_contribution_and_proof_intake(b2_ctx* ctx, const uint8_t* wire, uint64_t wire_len, const uint32_t* woff, uint32_t n,
                                          const uint32_t* position_validator, uint32_t committee_size, uint32_t subnet_count, uint64_t current_slot,
                                          const uint8_t* domains96, uint32_t target_aggregators, int32_t* status_out, uint32_t* root_id_out,
                                          uint8_t* roots32_out, uint32_t* n_roots_out, uint32_t* best_out, uint8_t* agg_bits_out,
                                          uint8_t* agg_sig96_out);
int b2_latest_messages_update_dev(b2_ctx* ctx, const uint32_t* d_members, const uint32_t* d_off, const uint8_t* d_bits,
                                  uint32_t bits_stride, const uint64_t* d_target_epoch, const uint32_t* d_block_idx,
                                  const uint8_t* d_accept, uint32_t n_agg, void* stream);
/* direct (un-propagated) vote weight per block in tree pre-order, u64[n_blocks]: the quantity that is summed across
 * GPUs (ncclAllReduce sum, u64) when validators are sharded; then b2_head_from_votes_dev finishes on every rank. */
int b2_vote_weights_dev(b2_ctx* ctx, uint64_t* d_votes_preorder, void* stream);
/* the same for the validators [v_begin, v_end) only: the get_head shard of one rank when ONE validator set is spread over the GPUs of
 * a box (BASELINE.json configs 4/5: N/8 validators per GPU, u64[n_blocks] all-reduce, head on every rank; pos-evolution.md:1102-1116) */
int b2_vote_weights_range_dev(b2_ctx* ctx, uint64_t v_begin, uint64_t v_end, uint64_t* d_votes_preorder, void* stream);
int b2_head_from_votes_dev(b2_ctx* ctx, uint64_t* d_votes_preorder, uint32_t justified_idx, int32_t boost_idx, uint64_t boost_score,
                           uint64_t* d_weight_out /* may be NULL */, uint32_t* d_head_idx_out, void* stream);
/* ---- get_head over ONE validator set spread over the GPUs of a box (BASELINE.json config 4; pos-evolution.md:1102-1116), one kernel
 * per rank with the all-reduce of the vote weights fused in over NVLink peer memory (no NCCL launch between scatter and tree):
 *   b2_fc_exchange_export  allocates this rank's exchange block (accumulators + flags, sized by the loaded tree) and returns its
 *                          64-byte CUDA IPC handle; the host layer all-gathers the handles of the ranks (any transport);
 *   b2_fc_exchange_open    maps every peer's block (handles64 = world x 64 bytes, in rank order);
 *   b2_get_head_multi      COLLECTIVE (every rank, same order): scatter the votes of this rank's validators [v_begin, v_end),
 *                          push the per-block sums into every rank's accumulator with 64-bit reductions over NVLink, flag
 *                          exchange, tree phase on the complete accumulator; returns the same head on every rank.
 * One process per GPU, at most 8 ranks, all on one NVLink/NVSwitch domain.  Re-export after b2_tree_load and after a b2_tree_add /
 * b2_tree_prune that changed the tree's size: until then b2_get_head_multi refuses (B2_EINVAL). */
int b2_fc_exchange_export(b2_ctx* ctx, uint8_t* handle64_out);
int b2_fc_exchange_open(b2_ctx* ctx, int rank, int world, const uint8_t* handles64);
int b2_get_head_multi(b2_ctx* ctx, uint64_t v_begin, uint64_t v_end, uint32_t justified_idx, int32_t boost_idx, uint64_t boost_score,
                      uint32_t* head_idx_out);
uint32_t b2_tree_size(b2_ctx* ctx);
/* profiling aid: SM-clock stamps of the phases of the context's last get_head (vote scatter of CTA 0, tree phases); u64[32].
 * Reading clears them: a slot that no call since the last read has written reads 0. */
int b2_debug_head_clocks(b2_ctx* ctx, uint64_t* out32);

/* ---- hash_tree_root of the beacon state's large fields (pos-evolution.md:338-374, checked at :423 and :1078).
 * b2_ssz_validators_load    builds the device node cache of List[Validator, 2^40] from n records of 121 bytes (the SSZ serialisation
 *                           of Validator, :36-45), n < 2^32 (0 allowed), and returns the list's root.  The cache holds 2C x 32 bytes,
 *                           C = next_pow2(max(n, 1)); it replaces the previous one only once complete.
 * b2_ssz_validators_update  replaces records idx[0..k) (strictly increasing, < n) in place, re-hashes those leaves and their paths to
 *                           the root, and returns the new root; k = 0 returns the current root.  B2_EINVAL, with nothing changed, on
 *                           unsorted, duplicate or out-of-range indices or without a loaded cache.  A registry that grows is re-loaded.
 * b2_ssz_chunks_root        the root of n_bytes of packed basic values: 32-byte chunks, the last zero-padded, merkleized to depth
 *                           limit_depth (n_bytes <= 32 * 2^limit_depth, limit_depth <= 64), then mix_in_length(root, length) when mix_in
 *                           is set.  The form of every basic-type list and vector of the state (balances, participation, inactivity
 *                           scores, randao_mixes, block_roots, state_roots, slashings).  Uses scratch only.
 * A context that never calls these allocates nothing for them. */
int b2_ssz_validators_load(b2_ctx* ctx, const uint8_t* rec121, uint64_t n, uint8_t* root32_out);
int b2_ssz_validators_update(b2_ctx* ctx, const uint32_t* idx, const uint8_t* rec121, uint64_t k, uint8_t* root32_out);
int b2_ssz_chunks_root(b2_ctx* ctx, const uint8_t* data, uint64_t n_bytes, uint32_t limit_depth, int mix_in, uint64_t length,
                       uint8_t* root32_out);

#ifdef __cplusplus
}
#endif
#endif /* B200POS_H */
