// aggintake.cuh -- one target epoch of aggregated attestations from gossip (SignedAggregateAndProof, the beacon_aggregate_and_proof topic
// of the upstream phase 0 p2p spec), checked on the device: decode, the stateless checks, the SSZ roots of the three signed messages,
// aggregator selection, the three signature checks through the existing verify paths, and the block-tree checks of the intake
// (intake.cuh).  The roots are __host__ __device__ so that tests/hostsim can run them on the CPU.  Included by b200pos.cu only.
//
//   k_api_parse       warp per item: the outer and inner containers, the nested Attestation (att_wire_parse), the bit row, checks 1-9,
//                     whether aggregator_index is a member of the committee; the member row; candidates counted per committee
//   k_api_data        thread per item: an insert-only hash table of the 128 data bytes, so that byte-equal data meet in one slot
//   k_api_roots       thread per item: data id, attestation signing root, block id; is_aggregator (12) and membership (13)
//   k_api_sets        thread per item: the slot and AggregateAndProof signing roots, the (signer, message, signature) sets of the two
//                     single-key checks, the bit row FastAggregateVerify reads, the tree checks (intake_tree_check)
//   FastAggregateVerify of every item (b2_fast_aggregate_verify_dev's path) and AggregateVerify of the 2n single-key sets
//   k_intake_scan / k_intake_scatter   the candidates bucketed by committee
//   k_api_committee   warp per committee: its candidates in list order, checks 10 and 11 against the ones accepted before, then 14-20
//   k_api_outsiders   thread per item: an item whose aggregator sits in another committee gets 11 if that aggregator was accepted earlier
//
// Wire form: SignedAggregateAndProof = [u32 offset of message = 100][signature 96][AggregateAndProof]; AggregateAndProof =
// [aggregator_index u64][u32 offset of aggregate = 108][selection_proof 96][Attestation].
#pragma once
#include "ssz.cuh"
#include "cores.cuh"

namespace b2 {

constexpr uint32_t API_OUTER_FIXED = 100;                            // SignedAggregateAndProof's fixed part
constexpr uint32_t API_INNER_FIXED = 108;                            // AggregateAndProof's fixed part
constexpr uint32_t API_ATT = API_OUTER_FIXED + API_INNER_FIXED;      // the nested Attestation's first byte
constexpr uint32_t API_PROOF = API_OUTER_FIXED + 12;                 // selection_proof

// the 32 bytes at p as digest words
HD void api_chunk_words(const uint8_t* p, uint32_t* c) {
#pragma unroll
    for (int i = 0; i < 8; i++) c[i] = ssz_be32(p + 4 * i);
}

// hash_tree_root(BLSSignature), a Vector[byte, 96]: three chunks padded to four
HD void api_sig_root(const uint8_t* sig96, uint32_t out[8]) {
    uint32_t in[16], a[8], b[8];
#pragma unroll
    for (int i = 0; i < 16; i++) in[i] = ssz_be32(sig96 + 4 * i);
    sha256_node(in, a);
#pragma unroll
    for (int i = 0; i < 8; i++) in[i] = ssz_be32(sig96 + 64 + 4 * i), in[8 + i] = 0;
    sha256_node(in, b);
    sha256_node_pair(a, b, out);
}

// hash_tree_root(Bitlist[2048]) of a bit row (delimiter removed, zero past nbits) of nbytes <= 256 bytes: 8 chunks, mix_in_length
HD void api_bitlist_root(const uint8_t* row, uint32_t nbytes, uint32_t nbits, uint32_t out[8]) {
    uint32_t l[4][8];
#pragma unroll 1
    for (int i = 0; i < 4; i++) {
        uint32_t in[16];
#pragma unroll
        for (int k = 0; k < 16; k++) {
            uint32_t w = 0;
#pragma unroll
            for (int j = 0; j < 4; j++) {
                const uint32_t b = 64 * i + 4 * k + j;
                w = w << 8 | (b < nbytes ? row[b] : 0u);
            }
            in[k] = w;
        }
        sha256_node(in, l[i]);
    }
    uint32_t a[8], b[8], r[8];
    sha256_node_pair(l[0], l[1], a);
    sha256_node_pair(l[2], l[3], b);
    sha256_node_pair(a, b, r);
    uint8_t le[8];
#pragma unroll
    for (int k = 0; k < 8; k++) le[k] = k < 4 ? (uint8_t)(nbits >> (8 * k)) : 0;
    ssz_u64_chunk(le, a);
    sha256_node_pair(r, a, out);
}

// hash_tree_root(Attestation): [aggregation_bits, data, signature] padded to four chunks
HD void api_attestation_root(const uint8_t* row, uint32_t nbytes, uint32_t nbits, const uint8_t* data_root32, const uint8_t* sig96, uint32_t out[8]) {
    uint32_t x[8], y[8], a[8], b[8];
    api_bitlist_root(row, nbytes, nbits, x);
    api_chunk_words(data_root32, y);
    sha256_node_pair(x, y, a);
    api_sig_root(sig96, x);
#pragma unroll
    for (int i = 0; i < 8; i++) y[i] = 0;
    sha256_node_pair(x, y, b);
    sha256_node_pair(a, b, out);
}

// hash_tree_root(AggregateAndProof): [aggregator_index, aggregate, selection_proof] padded to four chunks
HD void api_aggregate_and_proof_root(const uint8_t* aggregator_le8, const uint32_t att_root[8], const uint8_t* proof96, uint32_t out[8]) {
    uint32_t x[8], y[8], a[8], b[8];
    ssz_u64_chunk(aggregator_le8, x);
    sha256_node_pair(x, att_root, a);
    api_sig_root(proof96, x);
#pragma unroll
    for (int i = 0; i < 8; i++) y[i] = 0;
    sha256_node_pair(x, y, b);
    sha256_node_pair(a, b, out);
}

// compute_signing_root: hash_tree_root(SigningData(object_root, domain))
HD void api_signing_root(const uint32_t root[8], const uint8_t* domain32, uint8_t* out32) {
    uint32_t d[8], h[8];
    api_chunk_words(domain32, d);
    sha256_node_pair(root, d, h);
    ssz_store_root(h, out32);
}

// compute_signing_root(Slot(slot), domain) of a little-endian slot
HD void api_slot_signing_root(const uint8_t* slot_le8, const uint8_t* domain32, uint8_t* out32) {
    uint32_t c[8];
    ssz_u64_chunk(slot_le8, c);
    api_signing_root(c, domain32, out32);
}

// is_aggregator: bytes_to_uint64(hash(selection_proof)[0:8]) % max(1, committee_size // target) == 0 (target > 0)
HD bool api_is_aggregator(const uint8_t* proof96, uint32_t committee_size, uint32_t target) {
    sha256_ctx c;
    uint8_t d[32];
    sha256_init(c);
    sha256_update(c, proof96, 96);
    sha256_final(c, d);
    uint64_t v = 0;
#pragma unroll
    for (int k = 7; k >= 0; k--) v = v << 8 | d[k];
    const uint32_t m = committee_size / target;
    return v % (m > 1 ? m : 1u) == 0;
}

}  // namespace b2

#if defined(__CUDACC__)
#include "intake.cuh"

namespace b2 {

struct api_args {
    const uint8_t* wire;
    uint64_t wire_len;
    const uint32_t* woff;
    uint32_t n;
    const uint32_t* members;
    uint32_t committees_per_slot, slots_per_epoch, bits_stride, target_aggregators;
    uint64_t epoch, current_slot, propagation_range, n_val;
    intake_args T;      // committee layout (off, n_sig, bits_stride), epoch, and the device tree, as intake_row / intake_tree_check read them
    // scratch: per item, per hash-table slot, per committee, per validator, per single-key set
    uint32_t *fp, *slot_of, *dtab, *dmin, *acc, *accepted_by;
    uint32_t dtab_mask;
    uint8_t *incomm, *tst, *fbits;
    uint32_t *av_signer, *av_off;
    uint8_t *av_msg, *av_sig;
    const uint8_t *fav_ok, *av_ok;
    // outputs
    int32_t* status;
    uint32_t *committee, *data_id;
    uint8_t *bits, *sig96, *msg32;
    uint64_t* target_epoch;
    uint32_t *block_idx, *members_out, *item_off;
    intake_domain dom_att, dom_sel, dom_aap;
    uint32_t* guard;
};

__device__ __forceinline__ uint32_t api_le32(const uint8_t* p) {
    return (uint32_t)p[0] | (uint32_t)p[1] << 8 | (uint32_t)p[2] << 16 | (uint32_t)p[3] << 24;
}
__device__ __forceinline__ const uint8_t* api_item(const api_args& A, uint32_t a) { return A.wire + A.woff[a]; }
__device__ __forceinline__ uint64_t api_aggregator(const api_args& A, uint32_t a) { return intake_le64(api_item(A, a) + API_OUTER_FIXED); }

__global__ void __launch_bounds__(128) k_api_parse(api_args A) {
    const uint32_t a = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (a >= A.n) return;
    const uint32_t W = 8 * A.bits_stride;
    const uint32_t begin = A.woff[a], end = A.woff[a + 1];
    const uint8_t* w = A.wire + begin;
    const uint8_t* att = w + API_ATT;
    int32_t st = 1;
    uint32_t nbits = 0, c = VOTE_NONE, o0 = 0, size = 0, h = 0;
    uint64_t tgt = 0;
    bool in = false;
    if (begin <= end && end <= A.wire_len) {
        if (end - begin >= API_ATT && api_le32(w) == API_OUTER_FIXED && api_le32(w + API_OUTER_FIXED + 8) == API_INNER_FIXED)
            st = att_wire_parse(att, begin + API_ATT, end, A.bits_stride, W, nbits);
    } else if (lane == 0 && A.guard) {
        atomicOr(A.guard, (uint32_t)GUARD_BAD_ROW);
    }
    // the bit row with the delimiter cleared, zero past nbits; its population
    uint8_t* brow = A.bits + (uint64_t)a * A.bits_stride;
    uint32_t ones = 0;
    for (uint32_t k = lane; k < A.bits_stride; k += 32) {
        uint32_t x = 0;
        if (st == 0 && 8 * k < nbits) {
            x = att[B2_ATT_FIXED + k];
            if (8 * k + 8 > nbits) x &= (1u << (nbits & 7u)) - 1u;
        }
        brow[k] = (uint8_t)x;
        ones += __popc(x);
    }
    ones = __reduce_add_sync(B2_FULL_MASK, ones);
    for (uint32_t k = lane; k < 96; k += 32) A.sig96[96 * (uint64_t)a + k] = st == 0 ? att[132 + k] : 0;
    if (st == 0) {
        const uint8_t* d = att + 4;
        const uint8_t* dw = d + 4 * lane;      // a fingerprint of the 128 data bytes, as the intake's
        uint32_t x = ((uint32_t)dw[0] | (uint32_t)dw[1] << 8 | (uint32_t)dw[2] << 16 | (uint32_t)dw[3] << 24) ^ (lane * 0x9e3779b9u);
        x *= 0x85ebca6bu;
        h = __reduce_xor_sync(B2_FULL_MASK, x ^ (x >> 15));
        const uint64_t slot = intake_le64(d), index = intake_le64(d + 8), se = slot / A.slots_per_epoch;
        tgt = intake_le64(d + 88);
        if (index >= A.committees_per_slot) st = 4;
        else if (slot > A.current_slot || A.current_slot - slot > A.propagation_range) st = 5;
        else if (tgt != se) st = 6;
        else if (se != A.epoch) st = 7;
        else {
            c = (uint32_t)(slot - A.epoch * A.slots_per_epoch) * A.committees_per_slot + (uint32_t)index;
            if (!intake_row(A.T, c, o0, size)) {
                st = 8;      // a malformed committee row matches no length
                if (lane == 0 && A.guard) atomicOr(A.guard, (uint32_t)GUARD_BAD_ROW);
            } else if (nbits != size) {
                st = 8;
            } else if (ones == 0) {
                st = 9;
            } else {
                const uint64_t g = intake_le64(w + API_OUTER_FIXED);
                bool f = false;
                for (uint32_t j = lane; j < size; j += 32) f |= A.members[o0 + j] == g;
                in = __any_sync(B2_FULL_MASK, f);
            }
        }
    }
    // the member row the verification and update_latest_messages read: the committee, then zeros up to 8 * bits_stride
    uint32_t* mrow = A.members_out + (uint64_t)a * W;
    for (uint32_t j = lane; j < W; j += 32) mrow[j] = j < size ? A.members[o0 + j] : 0u;
    if (lane == 0) {
        A.item_off[a] = a * W;
        if (a == A.n - 1) A.item_off[A.n] = A.n * W;
        A.av_off[2 * a] = 2 * a;
        A.av_off[2 * a + 1] = 2 * a + 1;
        if (a == A.n - 1) A.av_off[2 * A.n] = 2 * A.n;
        A.status[a] = st;
        A.committee[a] = c;
        A.target_epoch[a] = st == 1 || st == 2 || st == 3 ? 0 : tgt;
        A.fp[a] = h;
        A.incomm[a] = in;
        A.T.comm[a] = st == 0 ? c : VOTE_NONE;
        if (st == 0) atomicAdd(&A.T.bucket[c], 1u);
    }
}

__device__ __forceinline__ bool api_decoded(int32_t st) { return st == 0 || st > 3; }

// thread per item: the first item whose data bytes claim a slot of the probe sequence owns it; the byte-equal ones join it
__global__ void __launch_bounds__(128) k_api_data(api_args A) {
    const uint32_t a = blockIdx.x * blockDim.x + threadIdx.x;
    if (a >= A.n) return;
    if (!api_decoded(A.status[a])) {
        A.slot_of[a] = VOTE_NONE;
        return;
    }
    const uint8_t* d = api_item(A, a) + API_ATT + 4;
    const uint32_t f = A.fp[a];
    uint32_t h = f & A.dtab_mask;
    for (;;) {      // the table holds at least 2n slots: a free one is always found
        const uint32_t o = atomicCAS(&A.dtab[h], VOTE_NONE, a);
        if (o == VOTE_NONE) break;
        if (A.fp[o] == f) {
            const uint8_t* e = api_item(A, o) + API_ATT + 4;
            bool eq = true;
            for (int k = 0; k < 128 && eq; k++) eq = d[k] == e[k];
            if (eq) break;
        }
        h = (h + 1) & A.dtab_mask;
    }
    A.slot_of[a] = h;
    atomicMin(&A.dmin[h], a);
}

__global__ void __launch_bounds__(64) k_api_roots(api_args A) {
    const uint32_t a = blockIdx.x * blockDim.x + threadIdx.x;
    if (a >= A.n) return;
    const int32_t st0 = A.status[a];
    const uint8_t* w = api_item(A, a);
    const uint8_t* d = w + API_ATT + 4;
    uint8_t* msg = A.msg32 + 32 * (uint64_t)a;
    if (!api_decoded(st0)) {
        for (int k = 0; k < 32; k++) msg[k] = 0;
        A.data_id[a] = VOTE_NONE;
        A.block_idx[a] = VOTE_NONE;
        return;
    }
    attestation_signing_root(d, A.dom_att.b, msg);
    A.data_id[a] = A.dmin[A.slot_of[a]];
    A.block_idx[a] = intake_find(A.T, d + 16);
    if (st0 == 0) {
        uint32_t o0, size;
        intake_row(A.T, A.committee[a], o0, size);      // a well-formed row: k_api_parse checked it
        if (!api_is_aggregator(w + API_PROOF, size, A.target_aggregators)) A.status[a] = 12;
        else if (!A.incomm[a]) A.status[a] = 13;
    }
}

// thread per item: the two single-key sets (selection proof, then the outer signature), the FastAggregateVerify bit row and the tree
// checks.  An item that failed before takes signer 0, zero messages and signatures and an empty row, so that nothing it carries reaches
// the pairing kernels.
__global__ void __launch_bounds__(64) k_api_sets(api_args A) {
    const uint32_t a = blockIdx.x * blockDim.x + threadIdx.x;
    if (a >= A.n) return;
    const bool go = A.status[a] == 0;
    const uint8_t* w = api_item(A, a);
    const uint8_t* d = w + API_ATT + 4;
    uint8_t* m0 = A.av_msg + 64 * (uint64_t)a;
    const uint8_t* row = A.bits + (uint64_t)a * A.bits_stride;
    if (go) {
        api_slot_signing_root(d, A.dom_sel.b, m0);
        uint8_t dr[32];
        uint32_t ar[8], pr[8];
        attestation_data_root(d, dr);
        uint32_t o0, size;
        intake_row(A.T, A.committee[a], o0, size);
        api_attestation_root(row, A.bits_stride, size, dr, w + API_ATT + 132, ar);
        api_aggregate_and_proof_root(w + API_OUTER_FIXED, ar, w + API_PROOF, pr);
        api_signing_root(pr, A.dom_aap.b, m0 + 32);
        uint32_t head = 0;
        A.tst[a] = (uint8_t)intake_tree_check(A.T, d, head);
    } else {
        for (int k = 0; k < 64; k++) m0[k] = 0;
    }
    const uint32_t signer = go ? (uint32_t)api_aggregator(A, a) : 0u;
    A.av_signer[2 * a] = signer;
    A.av_signer[2 * a + 1] = signer;
    uint8_t* s = A.av_sig + 192 * (uint64_t)a;
    for (int k = 0; k < 96; k++) {
        s[k] = go ? w[API_PROOF + k] : 0;
        s[96 + k] = go ? w[4 + k] : 0;
    }
    uint8_t* fb = A.fbits + (uint64_t)a * A.bits_stride;
    for (uint32_t k = 0; k < A.bits_stride; k++) fb[k] = go ? row[k] : 0;
}

// Warp per committee: its candidates (status 0, 12 or 13 so far) in list order.  An accepted item is added to acc[b0 ..] and, by its
// aggregator, to accepted_by (an accepted aggregator passed AggregateVerify, so it is a registry index).
__global__ void __launch_bounds__(32) k_api_committee(api_args A) {
    const uint32_t c = blockIdx.x, lane = threadIdx.x;
    const uint32_t b0 = A.T.bucket[c], m = A.T.bucket[c + 1] - b0, stride = A.bits_stride;
    uint32_t nacc = 0, last = 0;
    for (uint32_t i = 0; i < m; i++) {
        uint32_t best = VOTE_NONE;
        for (uint32_t j = lane; j < m; j += 32) {
            const uint32_t x = A.T.list[b0 + j];
            if ((i == 0 || x > last) && x < best) best = x;
        }
        const uint32_t a = __reduce_min_sync(B2_FULL_MASK, best);
        last = a;
        int32_t st = A.status[a];
        const uint32_t da = A.data_id[a];
        const uint64_t ga = api_aggregator(A, a);
        const uint8_t* ra = A.bits + (uint64_t)a * stride;
        bool shadow = false;      // check 10: an accepted item of the same data whose bits cover this item's
        for (uint32_t k = 0; k < nacc && !shadow; k++) {
            const uint32_t b = A.acc[b0 + k];
            if (A.data_id[b] != da) continue;
            const uint8_t* rb = A.bits + (uint64_t)b * stride;
            bool sub = true;
            for (uint32_t q = lane; q < stride; q += 32) sub &= (ra[q] & ~rb[q]) == 0;
            shadow = __all_sync(B2_FULL_MASK, sub);
        }
        bool same = false;        // check 11 inside the committee
        for (uint32_t k = lane; k < nacc; k += 32) same |= api_aggregator(A, A.acc[b0 + k]) == ga;
        same = __any_sync(B2_FULL_MASK, same);
        if (shadow) {
            st = 10;
        } else if (same) {
            st = 11;
        } else if (st == 0) {
            if (!A.av_ok[2 * a]) st = 14;
            else if (!A.av_ok[2 * a + 1]) st = 15;
            else if (!A.fav_ok[a]) st = 16;
            else if (A.tst[a]) st = 8 + A.tst[a];      // intake_tree_check's 9-12
            if (st == 0) {
                if (lane == 0) {
                    A.acc[b0 + nacc] = a;
                    if (ga < A.n_val) A.accepted_by[ga] = a;
                }
                nacc++;
            }
        }
        if (lane == 0) A.status[a] = st;
        __syncwarp();
    }
}

// thread per item: statuses 12 and 13 become 11 when the item's aggregator was accepted at an earlier list position (in any committee)
__global__ void __launch_bounds__(128) k_api_outsiders(api_args A) {
    const uint32_t a = blockIdx.x * blockDim.x + threadIdx.x;
    if (a >= A.n) return;
    const int32_t st = A.status[a];
    if (st != 12 && st != 13) return;
    const uint64_t g = api_aggregator(A, a);
    if (g < A.n_val && A.accepted_by[g] < a) A.status[a] = 11;
}

}  // namespace b2
#endif
