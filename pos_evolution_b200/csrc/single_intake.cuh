// single_intake.cuh -- one epoch of Electra's unaggregated attestations (SingleAttestation, the beacon_attestation_{subnet_id} topic of
// the upstream Electra p2p spec, EIP-7549), straight off the wire, turned into the inputs of the epoch pipeline's vote form.  Only the
// parse is new: it decodes the fixed-size container, applies checks 1-8 and finds the attester's committee position; everything after
// it is the phase 0 intake's (intake.cuh) unchanged.  Included by b200pos.cu only.
//
//   k_single_parse    warp per item: length, data.index, committee index, slot, subnet, target epoch, current slot, the attester's position
//                     (a warp search of its committee row); the data fingerprint; candidates counted per committee; the offset view
//   k_intake_scan, k_intake_scatter, k_intake_committee, k_intake_scan, k_intake_votes, k_intake_sigs   as for b2_attestation_intake
//
// Wire form: SingleAttestation = [committee_index u64][attester_index u64][AttestationData 128][signature 96], 240 bytes.
#pragma once
#include "intake.cuh"

namespace b2 {

constexpr uint32_t SINGLE_ATT_BYTES = 240;
// The phase 0 kernels read an item's data at woff + 4 and its signature at woff + 132; a SingleAttestation's sit at + 16 and + 144.
constexpr uint32_t SINGLE_VIEW_SHIFT = 12;

struct single_args {
    intake_args T;              // the arguments the reused kernels take; T.woff = view, which k_single_parse writes and never reads
    const uint32_t* woff;       // the items' own offsets, n_att + 1
    const uint32_t* members;    // committee c = members[off[c] .. off[c+1])
    const uint32_t* subnet;     // the subnet each item arrived on
    uint32_t subnet_count;
    uint32_t* view;             // out: woff[a] + SINGLE_VIEW_SHIFT, n_att entries
};

__global__ void __launch_bounds__(128) k_single_parse(single_args S) {
    const intake_args& A = S.T;
    const uint32_t a = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (a >= A.n_att) return;
    const uint32_t begin = S.woff[a], end = S.woff[a + 1];
    const uint8_t* w = A.wire + begin;
    int32_t st = 1;
    uint32_t c = VOTE_NONE, p = 0, h = 0;
    if (begin <= end && end <= A.wire_len) {
        if (end - begin == SINGLE_ATT_BYTES) st = 0;
    } else if (lane == 0 && A.guard) {
        atomicOr(A.guard, (uint32_t)GUARD_BAD_ROW);
    }
    if (st == 0) {
        const uint8_t* d = w + 16;
        // a fingerprint of the 128 data bytes, as the intake's
        const uint8_t* dw = d + 4 * lane;
        uint32_t x = ((uint32_t)dw[0] | (uint32_t)dw[1] << 8 | (uint32_t)dw[2] << 16 | (uint32_t)dw[3] << 24) ^ (lane * 0x9e3779b9u);
        x *= 0x85ebca6bu;
        h = __reduce_xor_sync(B2_FULL_MASK, x ^ (x >> 15));
        const uint64_t index = intake_le64(w), who = intake_le64(w + 8), slot = intake_le64(d), start = A.epoch * A.slots_per_epoch;
        if (intake_le64(d + 8) != 0) {
            st = 2;
        } else if (index >= A.committees_per_slot) {
            st = 3;
        } else if (slot - start >= A.slots_per_epoch) {      // (slot < start wraps)
            st = 4;
        } else {
            // compute_subnet_for_attestation with committee_index in data.index's place: slot % SLOTS_PER_EPOCH = slot - start here
            c = (uint32_t)(slot - start) * A.committees_per_slot + (uint32_t)index;
            if (c % S.subnet_count != S.subnet[a]) {
                st = 5;
            } else if (intake_le64(d + 88) != A.epoch) {
                st = 6;
            } else if (A.current_slot < slot + 1) {
                st = 7;
            } else {
                // the attester's position: the smallest one holding it (a malformed committee row has no members)
                uint32_t o0, size, at = VOTE_NONE;
                if (intake_row(A, c, o0, size))
                    for (uint32_t j = lane; j < size; j += 32)
                        if (S.members[o0 + j] == who) at = min(at, j);
                at = __reduce_min_sync(B2_FULL_MASK, at);
                if (at == VOTE_NONE) st = 8;
                else p = at;
            }
            if (st) c = VOTE_NONE;
        }
    }
    if (lane == 0) {
        A.status[a] = st;
        A.comm[a] = c;
        A.pos[a] = p;
        A.fp[a] = h;
        A.grp[a] = VOTE_NONE;
        S.view[a] = begin + SINGLE_VIEW_SHIFT;
        if (c != VOTE_NONE) atomicAdd(&A.bucket[c], 1u);
    }
}

}  // namespace b2
