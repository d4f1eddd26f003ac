// intake.cuh -- one epoch of unaggregated attestations, straight off the wire, turned into the inputs of the epoch pipeline's vote form
// (votes.cuh): process_attestation's checks (pos-evolution.md:724-730) and validate_on_attestation's (upstream fork-choice spec v1.2.0,
// :963-979) against the device block tree (tree.cuh), one attestation kept per committee position, the kept ones grouped by their
// AttestationData, and one signing root per distinct data.  Included by b200pos.cu only.
//
//   k_intake_parse      warp per attestation: container and delimiter (att_wire_parse), the single set bit, checks 1-8, committee and
//                       position; candidates are counted per committee
//   k_intake_scan       one CTA: bucket starts of the committees (exclusive scan of the counts, the total in bucket[n_committees])
//   k_intake_scatter    thread per candidate: its index into its committee's bucket
//   k_intake_committee  CTA per committee: the distinct data of its candidates (exact 128-byte comparison, a fingerprint first), the
//                       tree checks 9-12 once per distinct data, the position claims (smallest list index wins), vote numbering by the
//                       smallest position of each kept group
//   k_intake_scan       again: the vote counts into vote_off, the epoch's vote count in vote_off[n_committees]
//   k_intake_votes      thread per vote: data, signing root, epochs, block id
//   k_intake_sigs       CTA per committee: global vote ids and the kept signatures in committee order
#pragma once
#include "kernels.cuh"
#include "votes.cuh"

namespace b2 {

constexpr uint32_t INTAKE_THREADS = 256;

struct intake_domain {
    uint8_t b[32];
};

struct intake_args {
    const uint8_t* wire;
    uint64_t wire_len;
    const uint32_t* woff;
    uint32_t n_att;
    const uint32_t* off;                       // committee layout: committee c = member slots [off[c], off[c+1])
    uint32_t n_committees, committees_per_slot, slots_per_epoch, bits_stride;
    uint64_t n_sig, epoch, current_slot;
    // the device tree
    const uint8_t* root;
    const uint32_t* parent;
    const uint64_t* slot;
    const uint32_t* sorted;                    // block ids in (root, id) order
    uint32_t n_blocks;
    // scratch: per attestation, per committee, per bucket entry (a committee's candidates, then its distinct data), per member slot
    uint32_t *comm, *pos, *fp, *grp;
    uint32_t *bucket, *cursor, *nkept;
    uint32_t *list, *lead, *gstat, *gblk, *gmin, *vgrp;
    uint32_t* posatt;
    // outputs
    int32_t* status;
    uint32_t *vote, *vote_off;
    uint8_t* sig96;
    uint32_t max_votes;
    intake_domain domain;
    uint8_t *data128, *msg32;
    uint64_t *source_epoch, *target_epoch;
    uint32_t* block_idx;
    uint32_t* guard;
};

__device__ __forceinline__ uint64_t intake_le64(const uint8_t* p) {
    uint64_t v = 0;
#pragma unroll
    for (int i = 7; i >= 0; i--) v = v << 8 | p[i];
    return v;
}

// committee c's member slots [o0, o0 + size); false (size 0) for a row that is reversed, ends past n_sig or exceeds the bit row
__device__ __forceinline__ bool intake_row(const intake_args& A, uint32_t c, uint32_t& o0, uint32_t& size) {
    o0 = A.off[c];
    const uint32_t o1 = A.off[c + 1];
    const bool ok = o0 <= o1 && o1 <= A.n_sig && o1 - o0 <= 8 * A.bits_stride;
    size = ok ? o1 - o0 : 0;
    return ok;
}

// memcmp order of the 32-byte roots at x and y
__device__ __forceinline__ int intake_cmp32(const uint8_t* x, const uint8_t* y) {
    for (int i = 0; i < 32; i++)
        if (x[i] != y[i]) return x[i] < y[i] ? -1 : 1;
    return 0;
}

// the smallest block id whose root is r, or VOTE_NONE: a binary search of the root-sorted ids
__device__ uint32_t intake_find(const intake_args& A, const uint8_t* r) {
    uint32_t lo = 0, hi = A.n_blocks;
    while (lo < hi) {
        const uint32_t mid = (lo + hi) >> 1;
        if (intake_cmp32(A.root + 32ull * A.sorted[mid], r) < 0) lo = mid + 1;
        else hi = mid;
    }
    return lo < A.n_blocks && intake_cmp32(A.root + 32ull * A.sorted[lo], r) == 0 ? A.sorted[lo] : VOTE_NONE;
}

// checks 9-12 of one AttestationData d (128 bytes): 0 and the head block's id, or the failing status.  Block slots increase strictly
// along a chain and check 11 runs first, so the walk takes at most slots_per_epoch steps on a tree on_block builds; it is bounded by the
// tree's size all the same, because the slots come from the caller.
__device__ uint32_t intake_tree_check(const intake_args& A, const uint8_t* d, uint32_t& head) {
    const uint32_t h = intake_find(A, d + 16);
    if (h == VOTE_NONE) return 9;
    if (intake_find(A, d + 96) == VOTE_NONE) return 10;
    if (A.slot[h] > intake_le64(d)) return 11;
    const uint64_t start = A.epoch * A.slots_per_epoch;
    uint32_t b = h;
    for (uint32_t steps = 0; A.slot[b] > start; steps++) {
        if (b == 0 || steps >= A.n_blocks) return 12;      // the tree's root, still above start_slot(e): not the ancestor
        b = A.parent[b];
    }
    if (intake_cmp32(A.root + 32ull * b, d + 96) != 0) return 12;
    head = h;
    return 0;
}

// sorted[rank of (root, id)] = id
__global__ void k_intake_sorted(const uint32_t* __restrict__ rank, uint32_t n, uint32_t* __restrict__ sorted) {
    const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b < n) sorted[rank[b]] = b;
}

__global__ void __launch_bounds__(128) k_intake_parse(intake_args A) {
    const uint32_t a = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (a >= A.n_att) return;
    const uint32_t begin = A.woff[a], end = A.woff[a + 1];
    const uint8_t* w = A.wire + begin;
    int32_t st = 1;
    uint32_t nbits = 0, c = VOTE_NONE, p = 0, h = 0;
    if (begin <= end && end <= A.wire_len) {
        st = att_wire_parse(w, begin, end, A.bits_stride, 8 * A.bits_stride, nbits);
    } else if (lane == 0 && A.guard) {
        atomicOr(A.guard, (uint32_t)GUARD_BAD_ROW);
    }
    if (st == 0) {
        // the one set bit: the lanes scan the Bitlist's bytes with the delimiter cleared
        const uint32_t nbytes = end - begin - B2_ATT_FIXED;
        uint32_t ones = 0, at = 0;
        for (uint32_t k = lane; k < nbytes; k += 32) {
            uint32_t x = w[B2_ATT_FIXED + k];
            if (k == nbytes - 1) x &= (1u << (nbits & 7u)) - 1u;
            if (x) {
                ones += __popc(x);
                at = 8 * k + __ffs(x) - 1;
            }
        }
        ones = __reduce_add_sync(B2_FULL_MASK, ones);
        at = __reduce_max_sync(B2_FULL_MASK, at);
        // a fingerprint of the 128 data bytes (lane k mixes word k), so that the grouping compares bytes only where it matches
        const uint8_t* dw = w + 4 + 4 * lane;
        uint32_t x = ((uint32_t)dw[0] | (uint32_t)dw[1] << 8 | (uint32_t)dw[2] << 16 | (uint32_t)dw[3] << 24) ^ (lane * 0x9e3779b9u);
        x *= 0x85ebca6bu;
        h = __reduce_xor_sync(B2_FULL_MASK, x ^ (x >> 15));
        if (ones != 1) {
            st = 4;
        } else {
            const uint64_t slot = intake_le64(w + 4), index = intake_le64(w + 12), start = A.epoch * A.slots_per_epoch;
            if (slot - start >= A.slots_per_epoch || index >= A.committees_per_slot) {      // (slot < start wraps)
                st = 6;
            } else {
                uint32_t o0, size;
                c = (uint32_t)(slot - start) * A.committees_per_slot + (uint32_t)index;
                if (!intake_row(A, c, o0, size) || nbits != size) st = 5;      // a malformed committee row has no size to match
                else if (intake_le64(w + 92) != A.epoch) st = 7;
                else if (A.current_slot < slot + 1) st = 8;
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
        if (c != VOTE_NONE) atomicAdd(&A.bucket[c], 1u);
    }
}

// x[0 .. n) -> its exclusive scan and x[n] = the total (x holds n + 1 entries), in one CTA of 1024 threads; cursor (may be null)
// receives a copy of x[0 .. n)
__global__ void __launch_bounds__(1024) k_intake_scan(uint32_t* x, uint32_t n, uint32_t* cursor) {
    __shared__ uint32_t warp_tot[32];
    block_exclusive_scan(x, n, warp_tot);
    __syncthreads();
    if (cursor)
        for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) cursor[i] = x[i];
}

__global__ void k_intake_scatter(intake_args A) {
    const uint32_t a = blockIdx.x * blockDim.x + threadIdx.x;
    if (a >= A.n_att) return;
    const uint32_t c = A.comm[a];
    if (c != VOTE_NONE) A.list[atomicAdd(&A.cursor[c], 1u)] = a;
}

__device__ __forceinline__ uint32_t intake_block_min(uint32_t v, uint32_t* s_red) {
    v = __reduce_min_sync(B2_FULL_MASK, v);
    if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = v;
    __syncthreads();
    uint32_t r = VOTE_NONE;
    for (uint32_t w = 0; w < INTAKE_THREADS / 32; w++) r = min(r, s_red[w]);
    __syncthreads();
    return r;
}

// One CTA per committee.  Its candidates are list[b0 .. b0 + m); its distinct data k = 0 .. D-1 use the same range of lead / gstat /
// gblk / gmin, and its kept votes l the same range of vgrp (D <= m, kept votes <= D).
__global__ void __launch_bounds__(INTAKE_THREADS) k_intake_committee(intake_args A) {
    __shared__ uint32_t win[VOTES_MAX_MEMBERS];          // per position: the smallest list index claiming it
    __shared__ uint32_t first[VOTES_MAX_MEMBERS + 1];    // per position: 1 if it is its group's smallest kept position; then scanned,
                                                         // the total in first[size]
    __shared__ uint8_t ldata[128];
    __shared__ uint32_t s_red[INTAKE_THREADS / 32], warp_tot[32];
    const uint32_t c = blockIdx.x, tid = threadIdx.x;
    const uint32_t b0 = A.bucket[c], m = A.bucket[c + 1] - b0;
    uint32_t o0, size;
    if (!intake_row(A, c, o0, size) && tid == 0 && A.guard) atomicOr(A.guard, (uint32_t)GUARD_BAD_ROW);

    // the distinct data: the unassigned candidate with the smallest list index leads a new group, every candidate with its bytes joins it
    uint32_t D = 0;
    for (;;) {
        uint32_t best = VOTE_NONE;
        for (uint32_t j = tid; j < m; j += INTAKE_THREADS) {
            const uint32_t a = A.list[b0 + j];
            if (A.grp[a] == VOTE_NONE) best = min(best, a);
        }
        best = intake_block_min(best, s_red);
        if (best == VOTE_NONE) break;
        const uint8_t* ld = A.wire + A.woff[best] + 4;
        if (tid < 128) ldata[tid] = ld[tid];
        __syncthreads();
        const uint32_t lfp = A.fp[best];
        for (uint32_t j = tid; j < m; j += INTAKE_THREADS) {
            const uint32_t a = A.list[b0 + j];
            if (A.grp[a] != VOTE_NONE || A.fp[a] != lfp) continue;
            const uint8_t* d = A.wire + A.woff[a] + 4;
            bool eq = true;
            for (int k = 0; k < 128 && eq; k++) eq = d[k] == ldata[k];
            if (eq) A.grp[a] = D;
        }
        if (tid == 0) A.lead[b0 + D] = best;
        D++;
        __syncthreads();
    }
    // checks 9-12, once per distinct data
    for (uint32_t k = tid; k < D; k += INTAKE_THREADS) {
        uint32_t head = 0;
        A.gstat[b0 + k] = intake_tree_check(A, A.wire + A.woff[A.lead[b0 + k]] + 4, head);
        A.gblk[b0 + k] = head;
        A.gmin[b0 + k] = VOTE_NONE;
    }
    for (uint32_t p = tid; p < size; p += INTAKE_THREADS) win[p] = VOTE_NONE;
    __syncthreads();
    // claims: among the candidates whose data passed, the smallest list index takes the position; the others are duplicates
    for (uint32_t j = tid; j < m; j += INTAKE_THREADS) {
        const uint32_t a = A.list[b0 + j];
        if (A.gstat[b0 + A.grp[a]] == 0) atomicMin(&win[A.pos[a]], a);
    }
    __syncthreads();
    for (uint32_t j = tid; j < m; j += INTAKE_THREADS) {
        const uint32_t a = A.list[b0 + j], st = A.gstat[b0 + A.grp[a]];
        A.status[a] = st ? (int32_t)st : win[A.pos[a]] == a ? 0 : 13;
    }
    for (uint32_t p = tid; p < size; p += INTAKE_THREADS)
        if (win[p] != VOTE_NONE) atomicMin(&A.gmin[b0 + A.grp[win[p]]], p);
    __syncthreads();
    // votes: the kept groups in the order of their smallest position
    for (uint32_t p = tid; p < size; p += INTAKE_THREADS) first[p] = win[p] != VOTE_NONE && A.gmin[b0 + A.grp[win[p]]] == p ? 1u : 0u;
    __syncthreads();
    block_exclusive_scan(first, size, warp_tot);      // first[size] = the kept votes (size <= VOTES_MAX_MEMBERS)
    __syncthreads();
    for (uint32_t p = tid; p < size; p += INTAKE_THREADS) {
        const uint32_t a = win[p];
        uint32_t v = VOTE_NONE;
        if (a != VOTE_NONE) {
            const uint32_t g = A.grp[a], q = A.gmin[b0 + g];
            v = first[q];
            if (q == p) A.vgrp[b0 + v] = b0 + g;
        }
        A.vote[o0 + p] = v;      // the committee's local id; k_intake_sigs adds vote_off[c]
        A.posatt[o0 + p] = a;
    }
    if (tid == 0) {
        A.nkept[c] = first[size];
        A.vote_off[c] = max(first[size], 1u);      // a committee without a kept attestation has one placeholder vote
    }
}

// thread per vote row (the first max_votes votes of the epoch)
__global__ void __launch_bounds__(64) k_intake_votes(intake_args A) {
    const uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= A.max_votes || v >= A.vote_off[A.n_committees]) return;
    uint32_t lo = 0, hi = A.n_committees;      // vote_off[lo] <= v < vote_off[hi]
    while (hi - lo > 1) {
        const uint32_t mid = (lo + hi) >> 1;
        if (A.vote_off[mid] <= v) lo = mid;
        else hi = mid;
    }
    const uint32_t c = lo, l = v - A.vote_off[c];
    uint8_t d[128], o[32];
    uint32_t blk = 0;
    const bool kept = A.nkept[c] > 0;
    if (kept) {
        const uint32_t g = A.vgrp[A.bucket[c] + l];
        const uint8_t* src = A.wire + A.woff[A.lead[g]] + 4;
        for (int k = 0; k < 128; k++) d[k] = src[k];
        blk = A.gblk[g];
        attestation_signing_root(d, A.domain.b, o);
    } else {      // the placeholder: zero data, zero message
        for (int k = 0; k < 128; k++) d[k] = 0;
        for (int k = 0; k < 32; k++) o[k] = 0;
    }
    for (int k = 0; k < 128; k++) A.data128[128 * (uint64_t)v + k] = d[k];
    for (int k = 0; k < 32; k++) A.msg32[32 * (uint64_t)v + k] = o[k];
    A.source_epoch[v] = intake_le64(d + 48);
    A.target_epoch[v] = intake_le64(d + 88);
    A.block_idx[v] = blk;
}

// CTA per committee: the global vote id of every position, and its kept signature (zero where none is kept), word by word
__global__ void __launch_bounds__(INTAKE_THREADS) k_intake_sigs(intake_args A) {
    const uint32_t c = blockIdx.x;
    uint32_t o0, size;
    if (!intake_row(A, c, o0, size)) return;
    const uint32_t v0 = A.vote_off[c];
    for (uint32_t p = threadIdx.x; p < size; p += INTAKE_THREADS)
        if (A.vote[o0 + p] != VOTE_NONE) A.vote[o0 + p] += v0;
    uint32_t* out = reinterpret_cast<uint32_t*>(A.sig96) + (uint64_t)o0 * 24;
    for (uint32_t i = threadIdx.x; i < size * 24; i += INTAKE_THREADS) {
        const uint32_t p = i / 24, k = i - p * 24, a = A.posatt[o0 + p];
        uint32_t x = 0;
        if (a != VOTE_NONE) {
            const uint8_t* s = A.wire + A.woff[a] + 132 + 4 * k;
            x = (uint32_t)s[0] | (uint32_t)s[1] << 8 | (uint32_t)s[2] << 16 | (uint32_t)s[3] << 24;
        }
        out[i] = x;
    }
}

}  // namespace b2
