// syncmsg.cuh -- one slot of SyncCommitteeMessages from gossip (the container of pos-evolution.md:548-557; the sync_committee_{subnet_id}
// checks of the upstream Altair p2p spec), checked on the device, grouped by beacon_block_root, and summed into each subnet's
// SyncCommitteeContribution and each root's SyncAggregate (process_sync_committee_contributions of the upstream Altair validator spec).
// Included by b200pos.cu only, after aggintake.cuh (api_signing_root) and pack.cuh (k_pack_gather).
//
//   k_scm_index      one CTA: the committee's (validator << 32 | position) keys sorted by rank, so that the positions of a validator in a
//                    subnet are one binary search away; an entry >= n_validators gets validator 0xFFFFFFFF (matches nothing)
//   k_scm_parse      thread per item: decode, checks 1-4, the validator's first position in the item's subnet, and the single-key set
//                    (signer, signing root, signature) of check 6; an item that failed takes signer 0 and zero bytes
//   AggregateVerify of the n single-key sets (b2_aggregate_verify_dev's path)
//   k_scm_first      thread per item: per (validator, subnet), held at its first position, the first item in list order that verified
//   k_scm_accept     thread per item: checks 5 and 6; an accepted item claims its root in an insert-only table (exact 32-byte compare)
//   k_scm_number     one CTA: root ids by first occurrence in list order, the roots, n_roots; each accepted item's root id
//   k_scm_positions  thread per position: the accepted item of its validator on its subnet, and that item's root id
//   k_scm_rows       thread per (root, subnet): contribution row, present byte and segment size; thread per root: the aggregate row
//   k_intake_scan    the segment sizes into offsets
//   k_scm_gather     thread per position: the item of each set position, in (root, subnet, position) order; per root its first segment
//   k_g2_decompress, k_pack_gather, k_g2_segment_sum, k_g2_finish (unchanged): the contribution and aggregate signatures
//
// A root's positions are its subnets' positions, so in (root, subnet, position) order a root's aggregate is the run of its contributions:
// one gathered list serves both sums.  Each (validator, subnet) has at most one accepted item, so the list holds at most committee_size
// points; a validator holding k positions of a subnet appears k times.
//
// Wire form (144 bytes): slot u64 | beacon_block_root 32 | validator_index u64 | signature 96.
#pragma once
#include "aggintake.cuh"
#include "syncagg.cuh"

namespace b2 {

constexpr uint32_t SCM_WIRE = 144;
constexpr uint32_t SCM_ROOT = 8, SCM_VALIDATOR = 40, SCM_SIG = 48;

struct scm_args {
    const uint8_t* wire;
    uint64_t wire_len;
    const uint32_t* woff;
    uint32_t n;
    const uint32_t* subnet;
    const uint32_t* pos_val;
    uint32_t size, subnets, sub, sb, ab;      // committee_size, subnet_count, subcommittee size, contribution and aggregate row bytes
    uint64_t current_slot, n_val;
    intake_domain dom;
    // scratch: per position, per item, per hash-table slot, per (root, subnet) segment
    unsigned long long* keys;
    uint32_t *canon, *first, *pitem, *proot;
    uint32_t *signer, *pair_off;
    uint8_t *msg, *sig;
    const uint8_t* ok;
    uint32_t *slot_of, *rtab, *rmin, *rid;
    uint32_t rtab_mask;
    uint32_t *seg_off, *agg_off, *gsrc;
    // outputs
    int32_t* status;
    uint32_t *root_id, *n_roots;
    uint8_t *roots32, *cbits, *cpresent, *abits;
    uint32_t* guard;
};

__device__ __forceinline__ const uint8_t* scm_item(const scm_args& A, uint32_t a) { return A.wire + A.woff[a]; }

// the lowest position of validator v in subnet s, or VOTE_NONE
__device__ uint32_t scm_first_position(const scm_args& A, uint32_t v, uint32_t s) {
    const unsigned long long lo = (unsigned long long)v << 32 | (s * A.sub);
    uint32_t a = 0, b = A.size;
    while (a < b) {
        const uint32_t m = (a + b) >> 1;
        if (A.keys[m] < lo) a = m + 1;
        else b = m;
    }
    if (a == A.size) return VOTE_NONE;
    const unsigned long long k = A.keys[a];
    return (uint32_t)(k >> 32) == v && (uint32_t)k < (s + 1) * A.sub ? (uint32_t)k : VOTE_NONE;
}

__global__ void __launch_bounds__(1024) k_scm_index(scm_args A) {
    __shared__ unsigned long long k[B2_SYNC_MAX_SIZE];
    const uint32_t p = threadIdx.x;
    unsigned long long key = 0;
    if (p < A.size) {
        const uint32_t v = A.pos_val[p];
        const bool ok = v < A.n_val;
        if (!ok && A.guard) atomicOr(A.guard, (uint32_t)GUARD_BAD_INDEX);
        key = (unsigned long long)(ok ? v : VOTE_NONE) << 32 | p;
        k[p] = key;
    }
    __syncthreads();
    if (p < A.size) {
        uint32_t r = 0;      // the keys are distinct (their low words are): the rank is the sorted index
        for (uint32_t q = 0; q < A.size; q++) r += k[q] < key;
        A.keys[r] = key;
    }
}

__global__ void __launch_bounds__(128) k_scm_parse(scm_args A) {
    const uint32_t a = blockIdx.x * blockDim.x + threadIdx.x;
    if (a >= A.n) return;
    const uint32_t begin = A.woff[a], end = A.woff[a + 1];
    const uint8_t* w = A.wire + begin;
    int32_t st = 1;
    uint32_t pos = VOTE_NONE;
    uint64_t v = 0;
    if (begin > end || end > A.wire_len) {
        if (A.guard) atomicOr(A.guard, (uint32_t)GUARD_BAD_ROW);
    } else if (end - begin == SCM_WIRE) {
        const uint32_t s = A.subnet[a];
        v = intake_le64(w + SCM_VALIDATOR);
        if (intake_le64(w) != A.current_slot) st = 2;
        else if (v >= A.n_val) st = 3;      // n_val < 2^32: v fits a u32 from here on
        else if (s >= A.subnets || (pos = scm_first_position(A, (uint32_t)v, s)) == VOTE_NONE) st = 4;
        else st = 0;
    }
    const bool go = st == 0;
    A.status[a] = st;
    A.canon[a] = go ? pos : VOTE_NONE;
    A.signer[a] = go ? (uint32_t)v : 0u;
    A.pair_off[a] = a;
    if (a == A.n - 1) A.pair_off[A.n] = A.n;
    uint8_t* m = A.msg + 32 * (uint64_t)a;
    if (go) {
        uint32_t r[8];
        api_chunk_words(w + SCM_ROOT, r);
        api_signing_root(r, A.dom.b, m);
    } else {
        for (int k = 0; k < 32; k++) m[k] = 0;
    }
    uint8_t* s = A.sig + 96 * (uint64_t)a;
    for (int k = 0; k < 96; k++) s[k] = go ? w[SCM_SIG + k] : 0;
}

__global__ void __launch_bounds__(128) k_scm_first(scm_args A) {
    const uint32_t a = blockIdx.x * blockDim.x + threadIdx.x;
    if (a < A.n && A.status[a] == 0 && A.ok[a]) atomicMin(&A.first[A.canon[a]], a);
}

// Check 5 comes before the signature: an item after the accepted one of its (validator, subnet) is 5 whatever its signature; one before it
// (or with none accepted) and not verified is 6.
__global__ void __launch_bounds__(128) k_scm_accept(scm_args A) {
    const uint32_t a = blockIdx.x * blockDim.x + threadIdx.x;
    if (a >= A.n) return;
    A.slot_of[a] = VOTE_NONE;
    if (A.status[a] != 0) return;
    const uint32_t f = A.first[A.canon[a]];
    const int32_t st = f < a ? 5 : (A.ok[a] ? 0 : 6);
    A.status[a] = st;
    if (st) return;
    const uint8_t* r = scm_item(A, a) + SCM_ROOT;
    uint32_t h = ((uint32_t)r[0] | (uint32_t)r[1] << 8 | (uint32_t)r[2] << 16 | (uint32_t)r[3] << 24) ^ (uint32_t)r[31] << 24;
    h = (h * 0x9e3779b9u) >> 7;
    h &= A.rtab_mask;
    for (;;) {      // the table holds at least 2n slots: a free one is always found
        const uint32_t o = atomicCAS(&A.rtab[h], VOTE_NONE, a);
        if (o == VOTE_NONE) break;
        const uint8_t* e = scm_item(A, o) + SCM_ROOT;
        bool eq = true;
        for (int k = 0; k < 32 && eq; k++) eq = r[k] == e[k];
        if (eq) break;
        h = (h + 1) & A.rtab_mask;
    }
    A.slot_of[a] = h;
    atomicMin(&A.rmin[h], a);
}

// one CTA over the items in list order: the first accepted item of each root leads it, the leaders are numbered in list order
__global__ void __launch_bounds__(1024) k_scm_number(scm_args A) {
    __shared__ uint32_t wsum[32];
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nw = blockDim.x >> 5;
    uint32_t base = 0;
    for (uint32_t c0 = 0; c0 < A.n; c0 += blockDim.x) {
        const uint32_t a = c0 + tid;
        const uint32_t h = a < A.n ? A.slot_of[a] : VOTE_NONE;
        const bool lead = h != VOTE_NONE && A.rmin[h] == a;
        const unsigned m = __ballot_sync(B2_FULL_MASK, lead);
        if (lane == 0) wsum[warp] = __popc(m);
        __syncthreads();
        uint32_t before = base, total = 0;
        for (uint32_t q = 0; q < nw; q++) {
            before += q < warp ? wsum[q] : 0u;
            total += wsum[q];
        }
        if (lead) {
            const uint32_t id = before + __popc(m & ((1u << lane) - 1u));
            A.rid[a] = id;
            const uint8_t* r = scm_item(A, a) + SCM_ROOT;
            for (int k = 0; k < 32; k++) A.roots32[32 * (uint64_t)id + k] = r[k];
        }
        base += total;
        __syncthreads();
    }
    if (tid == 0) *A.n_roots = base;
    for (uint32_t a = tid; a < A.n; a += blockDim.x) {
        const uint32_t h = A.slot_of[a];
        A.root_id[a] = h == VOTE_NONE ? VOTE_NONE : A.rid[A.rmin[h]];
    }
    for (uint64_t b = 32 * (uint64_t)base + tid; b < 32 * (uint64_t)A.n; b += blockDim.x) A.roots32[b] = 0;
}

__global__ void __launch_bounds__(128) k_scm_positions(scm_args A) {
    const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= A.size) return;
    const uint32_t v = A.pos_val[p];
    uint32_t item = VOTE_NONE;
    if (v < A.n_val) item = A.first[scm_first_position(A, v, p / A.sub)];      // p itself is a position of v in its subnet
    A.pitem[p] = item;
    A.proot[p] = item == VOTE_NONE ? VOTE_NONE : A.root_id[item];
}

// threads [0, n * subnets): contribution (root t / subnets, subnet t % subnets); threads [n * subnets, n * (subnets + 1)): the aggregate row of
// root t - n * subnets.  Rows of roots >= n_roots come out zero (no position names them).
__global__ void __launch_bounds__(128) k_scm_rows(scm_args A) {
    const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x, nc = (uint64_t)A.n * A.subnets;
    if (t < nc) {
        const uint32_t r = (uint32_t)(t / A.subnets), p0 = (uint32_t)(t % A.subnets) * A.sub;
        uint8_t* row = A.cbits + t * A.sb;
        uint32_t c = 0;
        for (uint32_t j = 0; j < A.sb; j++) {
            uint32_t x = 0;
            for (uint32_t i = 0; i < 8; i++) {
                const uint32_t q = 8 * j + i;
                if (q < A.sub && A.proot[p0 + q] == r) x |= 1u << i;
            }
            row[j] = (uint8_t)x;
            c += __popc(x);
        }
        A.cpresent[t] = c != 0;
        A.seg_off[t] = c;
    } else if (t < nc + A.n) {
        const uint32_t r = (uint32_t)(t - nc);
        uint8_t* row = A.abits + (uint64_t)r * A.ab;
        for (uint32_t j = 0; j < A.ab; j++) {
            uint32_t x = 0;
            for (uint32_t i = 0; i < 8; i++) {
                const uint32_t q = 8 * j + i;
                if (q < A.size && A.proot[q] == r) x |= 1u << i;
            }
            row[j] = (uint8_t)x;
        }
    }
}

// threads [0, size): each set position's item at its place in (root, subnet, position) order; threads [0, n]: agg_off[r] = seg_off[r * subnets]
__global__ void __launch_bounds__(128) k_scm_gather(scm_args A) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t <= A.n) A.agg_off[t] = A.seg_off[(uint64_t)t * A.subnets];
    if (t >= A.size) return;
    const uint32_t r = A.proot[t];
    if (r == VOTE_NONE) return;
    const uint32_t s = t / A.sub;
    uint32_t rank = 0;
    for (uint32_t q = s * A.sub; q < t; q++) rank += A.proot[q] == r;
    A.gsrc[A.seg_off[(uint64_t)r * A.subnets + s] + rank] = A.pitem[t];
}

}  // namespace b2
