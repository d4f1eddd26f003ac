// blockatt.cuh -- process_attestation (pos-evolution.md:722-754) for the attestations of a run of blocks of one chain in one epoch e,
// block-atomic as on_block's state_transition (:1008-1009): the blocks before the first invalid one are applied in order, nothing of
// that block or of a later one.  Within one epoch nothing process_attestation reads changes between blocks except the participation
// tables it writes, and the flag scatter is order-exact over a whole batch (k_part_phase1-3), so one call gives the state the spec
// gives block by block.  Included by b200pos.cu only.
//
//   k_ba_parse     warp per attestation: its block (block_off), the container (att_wire_parse), checks 1-9 against the block's slot,
//                  the committees of e-1 and e, the justified checkpoints and the chain's roots; the participation flag mask (:733);
//                  the zero-padded member row, bit row and signature FastAggregateVerify reads; the data and the attester domain of
//                  its target epoch
//   k_signing_roots (kernels.cuh) thread per attestation: compute_signing_root(data, domain)
//   FastAggregateVerify of every attestation (b2_fast_aggregate_verify_dev's path)
//   k_ba_blocks    one CTA: checks 10-11 folded into the statuses, each block's first failing attestation, the first invalid block,
//                  the accept masks of the two participation tables
//   k_part_phase1-3 (kernels.cuh) over the accept mask of the current table, then of the previous one
//   k_ba_rewards   warp per block: each attestation's numerator, and the block's sum of numerator // 448 (:752-754)
#pragma once
#include "intake.cuh"

namespace b2 {

constexpr uint32_t BA_BLOCKS_THREADS = 1024;
// (WEIGHT_DENOMINATOR - PROPOSER_WEIGHT) * WEIGHT_DENOMINATOR // PROPOSER_WEIGHT (:752)
constexpr unsigned long long BA_REWARD_DENOMINATOR = (64ull - 8ull) * 64ull / 8ull;

struct ba_checkpoints {
    uint8_t b[80];      // previous_justified_checkpoint, then current_justified_checkpoint: epoch u64 LE || root
};

struct ba_args {
    const uint8_t* wire;
    uint64_t wire_len;
    const uint32_t* woff;
    uint32_t n;
    const uint32_t* block_off;                 // block b = attestations [block_off[b], block_off[b+1])
    const uint64_t* block_slot;                // e = block_slot[0] / slots_per_epoch
    uint32_t n_blocks;
    const uint32_t* members;
    intake_args T;                             // committee layout (off, n_sig, bits_stride) as intake_row reads it
    uint32_t cps_prev, cps_cur, slots_per_epoch, bits_stride, min_delay, isqrt_spe;
    const uint8_t* chain_roots;                // u8[2 * slots_per_epoch][32]: slot s at s + slots_per_epoch - start(e)
    ba_checkpoints justified;
    intake_domain dom[2];                      // attester domains of e - 1 and e
    // scratch: per attestation its block (VOTE_NONE: in no block's row), whether its target is e, the FastAggregateVerify verdict,
    // the accept masks (table 0, then table 1) and the numerators of table 1
    uint32_t* blk_of;
    uint8_t *cur, *fav_ok, *accept;
    unsigned long long* num1;
    // FastAggregateVerify inputs, and the data and domain rows k_signing_roots reads
    uint8_t *bits, *sig96, *data128, *dom32;
    uint32_t *members_out, *item_off;
    // outputs
    int32_t* status;
    uint8_t* flag_mask;
    unsigned long long* numerator;
    int32_t* block_status;
    uint32_t* block_first;
    unsigned long long* block_reward;
    uint32_t* n_applied;
    uint32_t* guard;
};

// the block whose row holds attestation a, or VOTE_NONE: the last b with block_off[b] <= a, if a < block_off[b+1] <= n
__device__ __forceinline__ uint32_t ba_block_of(const ba_args& A, uint32_t a) {
    uint32_t lo = 0, hi = A.n_blocks;
    while (lo < hi) {
        const uint32_t mid = (lo + hi) >> 1;
        if (A.block_off[mid] <= a) lo = mid + 1;
        else hi = mid;
    }
    if (lo == 0) return VOTE_NONE;
    const uint32_t b = lo - 1;
    return A.block_off[b] <= a && a < A.block_off[b + 1] && A.block_off[b + 1] <= A.n ? b : VOTE_NONE;
}

// 32 bytes equal, one byte per lane (the whole warp calls it)
__device__ __forceinline__ bool ba_eq32(const uint8_t* x, const uint8_t* y, uint32_t lane) { return __all_sync(B2_FULL_MASK, x[lane] == y[lane]); }

__global__ void __launch_bounds__(128) k_ba_parse(ba_args A) {
    const uint32_t a = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (a >= A.n) return;
    const uint32_t W = 8 * A.bits_stride, spe = A.slots_per_epoch;
    const uint64_t e = A.block_slot[0] / spe, start = e * spe;
    const uint32_t b = ba_block_of(A, a);
    const uint32_t begin = A.woff[a], end = A.woff[a + 1];
    const uint8_t* w = A.wire + begin;
    int32_t st = 1;
    uint32_t nbits = 0, o0 = 0, size = 0, mask = 0;
    bool cur = false;
    if (b != VOTE_NONE && begin <= end && end <= A.wire_len) st = att_wire_parse(w, begin, end, A.bits_stride, W, nbits);
    else if (lane == 0 && A.guard) atomicOr(A.guard, (uint32_t)GUARD_BAD_ROW);
    uint32_t ones = 0;
    for (uint32_t k = lane; st == 0 && 8 * k < nbits; k += 32) {
        uint32_t x = w[B2_ATT_FIXED + k];
        if (8 * k + 8 > nbits) x &= (1u << (nbits & 7u)) - 1u;
        ones += __popc(x);
    }
    ones = __reduce_add_sync(B2_FULL_MASK, ones);
    if (st == 0) {
        const uint8_t* d = w + 4;
        const uint64_t slot = intake_le64(d), index = intake_le64(d + 8), tgt = intake_le64(d + 88), bslot = A.block_slot[b];
        cur = tgt == e;
        const uint32_t cps = cur ? A.cps_cur : A.cps_prev;
        if (!cur && (e == 0 || tgt != e - 1)) st = 4;
        else if (tgt != slot / spe) st = 5;
        else if (slot + A.min_delay > bslot || bslot > slot + spe) st = 6;
        else if (index >= cps) st = 7;
        else {
            // index < cps and slot - start(tgt) < spe: c < (cps_prev + cps_cur) * spe, the committee count
            const uint32_t c = (cur ? A.cps_prev * spe : 0u) + (uint32_t)(slot - tgt * spe) * cps + (uint32_t)index;
            const uint8_t* J = A.justified.b + (cur ? 40 : 0);
            bool src = true;
            for (uint32_t k = lane; k < 40; k += 32) src &= d[48 + k] == J[k];
            src = __all_sync(B2_FULL_MASK, src);
            if (!intake_row(A.T, c, o0, size)) {
                st = 8;      // a malformed committee row matches no length
                if (lane == 0 && A.guard) atomicOr(A.guard, (uint32_t)GUARD_BAD_ROW);
            } else if (nbits != size) {
                st = 8;
            } else if (!src) {
                st = 9;
            } else {
                // get_block_root(target epoch) = the root at start(tgt); get_block_root_at_slot(data.slot); slot >= start(e - 1) by check 5
                const bool target = ba_eq32(d + 96, A.chain_roots + 32ull * (cur ? spe : 0u), lane);
                const bool head = ba_eq32(d + 16, A.chain_roots + 32ull * (slot + spe - start), lane);
                const uint64_t delay = bslot - slot;
                mask = (delay <= A.isqrt_spe ? 1u : 0u) | (target && delay <= spe ? 2u : 0u) | (target && head && delay == A.min_delay ? 4u : 0u);
                if (ones == 0) st = 10;
            }
        }
    }
    // what FastAggregateVerify and the flag scatter read: the bit row, the signature and the committee, zero padded; all zero unless
    // the attestation passed checks 1-10
    const bool go = st == 0;
    uint8_t* brow = A.bits + (uint64_t)a * A.bits_stride;
    for (uint32_t k = lane; k < A.bits_stride; k += 32) {
        uint32_t x = 0;
        if (go && 8 * k < nbits) {
            x = w[B2_ATT_FIXED + k];
            if (8 * k + 8 > nbits) x &= (1u << (nbits & 7u)) - 1u;
        }
        brow[k] = (uint8_t)x;
    }
    for (uint32_t k = lane; k < 96; k += 32) A.sig96[96 * (uint64_t)a + k] = go ? w[132 + k] : 0;
    for (uint32_t k = lane; k < 128; k += 32) A.data128[128 * (uint64_t)a + k] = go ? w[4 + k] : 0;
    A.dom32[32 * (uint64_t)a + lane] = go ? A.dom[cur].b[lane] : 0;
    uint32_t* mrow = A.members_out + (uint64_t)a * W;
    for (uint32_t j = lane; j < W; j += 32) mrow[j] = go && j < size ? A.members[o0 + j] : 0u;
    if (lane == 0) {
        A.item_off[a] = a * W;
        if (a == A.n - 1) A.item_off[A.n] = A.n * W;
        A.status[a] = st;
        A.flag_mask[a] = (uint8_t)mask;
        A.blk_of[a] = b;
        A.cur[a] = cur;
    }
}

// One CTA.  A block is invalid when its row is malformed (reversed, past n, a slot outside e or not above the previous block's, or an
// attestation of its row that ba_block_of gave to another block: B2_GUARD_BAD_ROW) or when it holds an attestation with a nonzero status.
// An attestation that passed the parse's checks and failed FastAggregateVerify gets fav_status (11; 13 in the Electra form).
__global__ void __launch_bounds__(BA_BLOCKS_THREADS) k_ba_blocks(ba_args A, int32_t fav_status) {
    __shared__ uint32_t first_bad;
    if (threadIdx.x == 0) first_bad = A.n_blocks;
    for (uint32_t a = threadIdx.x; a < A.n; a += blockDim.x)
        if (A.status[a] == 0 && !A.fav_ok[a]) A.status[a] = fav_status;
    __syncthreads();
    const uint64_t spe = A.slots_per_epoch, e = A.block_slot[0] / spe;
    for (uint32_t b = threadIdx.x; b < A.n_blocks; b += blockDim.x) {
        const uint32_t b0 = A.block_off[b], b1 = A.block_off[b + 1];
        const uint64_t s = A.block_slot[b];
        bool bad = b0 > b1 || b1 > A.n || s / spe != e || (b > 0 && s <= A.block_slot[b - 1]);
        uint32_t f = VOTE_NONE;
        for (uint32_t a = b0; !bad && f == VOTE_NONE && a < b1; a++) {
            if (A.blk_of[a] != b) bad = true;
            else if (A.status[a] != 0) f = a - b0;
        }
        if (bad) {
            f = VOTE_NONE;
            if (A.guard) atomicOr(A.guard, (uint32_t)GUARD_BAD_ROW);
        }
        A.block_first[b] = f;
        A.block_status[b] = bad || f != VOTE_NONE;
        if (bad || f != VOTE_NONE) atomicMin(&first_bad, b);
    }
    __syncthreads();
    const uint32_t fb = first_bad;
    for (uint32_t b = threadIdx.x; b < A.n_blocks; b += blockDim.x)
        if (b > fb && A.block_status[b] == 0) A.block_status[b] = 2;
    if (threadIdx.x == 0) *A.n_applied = fb;
    for (uint32_t a = threadIdx.x; a < A.n; a += blockDim.x) {
        const bool ok = A.blk_of[a] < fb && A.status[a] == 0;
        A.accept[a] = ok && A.cur[a];
        A.accept[A.n + a] = ok && !A.cur[a];
    }
}

// warp per block: numerator = the current table's (already in `numerator`) + the previous table's; the block's proposer reward
__global__ void __launch_bounds__(128) k_ba_rewards(ba_args A) {
    const uint32_t b = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (b >= A.n_blocks) return;
    const uint32_t b0 = A.block_off[b], b1 = A.block_off[b + 1];
    unsigned long long sum = 0;
    if (b0 <= b1 && b1 <= A.n)
        for (uint32_t a = b0 + lane; a < b1; a += 32)
            if (A.blk_of[a] == b) {      // one writer per attestation, whatever the rows
                const unsigned long long v = A.numerator[a] + A.num1[a];
                A.numerator[a] = v;
                sum += v / BA_REWARD_DENOMINATOR;
            }
#pragma unroll
    for (int d = 16; d >= 1; d >>= 1) sum += __shfl_down_sync(B2_FULL_MASK, sum, d);
    if (lane == 0) A.block_reward[b] = sum;
}

}  // namespace b2
