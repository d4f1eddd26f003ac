// synccontrib.cuh -- one slot of SignedContributionAndProof from gossip (the sync_committee_contribution_and_proof topic of the upstream
// Altair p2p spec), checked on the device, and each beacon_block_root's SyncAggregate built from its best contribution per subnet
// (process_sync_committee_contributions of the upstream Altair validator spec).  The SSZ roots are __host__ __device__ so that tests/hostsim
// can run them on the CPU.  Included by b200pos.cu only, after syncmsg.cuh (k_scm_index, scm_first_position, k_scm_number).
//
//   k_scm_index      (unchanged) the committee's (validator << 32 | position) keys sorted, so a validator's positions in a subnet are one
//                    binary search away
//   k_scc_parse      thread per item: decode, checks 1-7, the three signing roots, the two single-key sets (selection proof, outer
//                    signature), the member and bit rows and message of the contribution's FastAggregateVerify, and the item's root in an
//                    insert-only table (exact 32-byte compare); an item that failed takes signer 0, zero bytes and an empty row
//   AggregateVerify of the 2n single-key sets, FastAggregateVerify of the n contributions (the intakes' paths)
//   k_scc_order      warp per subnet: its candidates in list order; checks 8 and 9 against the items it accepted before, then 10-12
//   k_scc_claim      thread per item: an accepted item claims the first-occurrence slot of its root
//   k_scm_number     (unchanged) root ids by first accepted occurrence, the roots, n_roots, each accepted item's root id
//   k_scc_best       thread per item: per (root, subnet) the accepted item with the most bits, ties to the smaller list index
//   k_scc_rows       thread per root: best, the aggregate's bit row and the number of present subnets; k_intake_scan -> segment offsets
//   k_scc_gather     thread per root: its best items in subnet order
//   k_g2_decompress, k_pack_gather, k_g2_segment_sum, k_g2_finish (unchanged): each root's aggregate signature
//
// Wire form (344 + ceil(sub / 8) bytes, every field fixed): SignedContributionAndProof = ContributionAndProof | signature 96;
// ContributionAndProof = aggregator_index u64 | SyncCommitteeContribution | selection_proof 96; SyncCommitteeContribution = slot u64 |
// beacon_block_root 32 | subcommittee_index u64 | aggregation_bits Bitvector[sub] | signature 96.
#pragma once
#include "aggintake.cuh"

namespace b2 {

constexpr uint32_t SCC_FIXED = 344;                                    // every field but the Bitvector
constexpr uint32_t SCC_SLOT = 8, SCC_ROOT = 16, SCC_INDEX = 48, SCC_BITS = 56;
HD uint32_t scc_sig(uint32_t sb) { return SCC_BITS + sb; }         // the contribution's signature
HD uint32_t scc_proof(uint32_t sb) { return SCC_BITS + sb + 96; }  // selection_proof
HD uint32_t scc_outer(uint32_t sb) { return SCC_BITS + sb + 192; } // the outer signature

// hash_tree_root(Bitvector[sub]) of its sb = ceil(sub / 8) <= 128 bytes: ceil(sb / 32) chunks padded to a power of two, no length mix-in
HD void scc_bitvector_root(const uint8_t* row, uint32_t sb, uint32_t out[8]) {
    uint32_t l[4][8];
#pragma unroll
    for (uint32_t i = 0; i < 4; i++)
#pragma unroll
        for (uint32_t k = 0; k < 8; k++) {
            uint32_t w = 0;
#pragma unroll
            for (uint32_t j = 0; j < 4; j++) {
                const uint32_t b = 32 * i + 4 * k + j;
                w = w << 8 | (b < sb ? row[b] : 0u);
            }
            l[i][k] = w;
        }
    const uint32_t chunks = (sb + 31) / 32;
    if (chunks <= 1) {
#pragma unroll
        for (int k = 0; k < 8; k++) out[k] = l[0][k];
    } else if (chunks == 2) {
        sha256_node_pair(l[0], l[1], out);
    } else {
        uint32_t a[8], b[8];
        sha256_node_pair(l[0], l[1], a);
        sha256_node_pair(l[2], l[3], b);
        sha256_node_pair(a, b, out);
    }
}

// hash_tree_root(SyncCommitteeContribution) of its wire bytes c: [slot, beacon_block_root, subcommittee_index, aggregation_bits, signature]
// padded to eight chunks
HD void scc_contribution_root(const uint8_t* c, uint32_t sb, uint32_t out[8]) {
    uint32_t x[8], y[8], a[8], b[8];
    ssz_u64_chunk(c, x);
    api_chunk_words(c + 8, y);
    sha256_node_pair(x, y, a);
    ssz_u64_chunk(c + 40, x);
    scc_bitvector_root(c + 48, sb, y);
    sha256_node_pair(x, y, b);
    sha256_node_pair(a, b, out);      // the left half
    api_sig_root(c + 48 + sb, x);
#pragma unroll
    for (int i = 0; i < 8; i++) y[i] = 0;
    sha256_node_pair(x, y, a);        // [signature, 0]
    sha256_node_pair(y, y, x);        // [0, 0]
    sha256_node_pair(a, x, b);        // the right half
    sha256_node_pair(out, b, a);
#pragma unroll
    for (int i = 0; i < 8; i++) out[i] = a[i];
}

// hash_tree_root(ContributionAndProof) of its wire bytes m: [aggregator_index, contribution, selection_proof] padded to four chunks
HD void scc_contribution_and_proof_root(const uint8_t* m, uint32_t sb, uint32_t out[8]) {
    uint32_t x[8], y[8], a[8], b[8];
    ssz_u64_chunk(m, x);
    scc_contribution_root(m + SCC_SLOT, sb, y);
    sha256_node_pair(x, y, a);
    api_sig_root(m + scc_proof(sb), x);
#pragma unroll
    for (int i = 0; i < 8; i++) y[i] = 0;
    sha256_node_pair(x, y, b);
    sha256_node_pair(a, b, out);
}

// hash_tree_root(SyncAggregatorSelectionData(slot, subcommittee_index)) of two little-endian u64: one node
HD void scc_selection_data_root(const uint8_t* slot_le8, const uint8_t* index_le8, uint32_t out[8]) {
    uint32_t x[8], y[8];
    ssz_u64_chunk(slot_le8, x);
    ssz_u64_chunk(index_le8, y);
    sha256_node_pair(x, y, out);
}

// SHA-256 compression of one block w[16] (big-endian words; the schedule is built in place) into the state h[8]
HD void scc_sha_compress(uint32_t h[8], uint32_t w[16]) {
    uint32_t s[8];
#pragma unroll
    for (int i = 0; i < 8; i++) s[i] = h[i];
#pragma unroll
    for (int i = 0; i < 64; i++) {
        if (i >= 16) {
            const uint32_t w15 = w[(i - 15) & 15], w2 = w[(i - 2) & 15];
            w[i & 15] += (sha_rotr(w15, 7) ^ sha_rotr(w15, 18) ^ (w15 >> 3)) + w[(i - 7) & 15] + (sha_rotr(w2, 17) ^ sha_rotr(w2, 19) ^ (w2 >> 10));
        }
        sha_round(s, sha_k(i) + w[i & 15]);
    }
#pragma unroll
    for (int i = 0; i < 8; i++) h[i] += s[i];
}

// is_sync_committee_aggregator: bytes_to_uint64(hash(selection_proof)[0:8]) % max(1, sub // target) == 0 (target > 0).  The hash of the
// 96 bytes is two compressions in registers (api_is_aggregator's streaming context would put a buffer on the stack).
HD bool scc_is_aggregator(const uint8_t* proof96, uint32_t sub, uint32_t target) {
    uint32_t h[8] = {0x6a09e667, 0xbb67ae85, 0x3c6ef372, 0xa54ff53a, 0x510e527f, 0x9b05688c, 0x1f83d9ab, 0x5be0cd19}, w[16];
#pragma unroll
    for (int i = 0; i < 16; i++) w[i] = ssz_be32(proof96 + 4 * i);
    scc_sha_compress(h, w);
#pragma unroll
    for (int i = 0; i < 16; i++) w[i] = i < 8 ? ssz_be32(proof96 + 64 + 4 * i) : i == 8 ? 0x80000000u : i == 15 ? 768u : 0u;
    scc_sha_compress(h, w);
    uint64_t v = 0;      // the digest's first 8 bytes, little-endian: bytes 0-3 are h[0]'s, most significant first
#pragma unroll
    for (int k = 0; k < 4; k++) v |= (uint64_t)((h[0] >> (24 - 8 * k)) & 0xffu) << (8 * k) | (uint64_t)((h[1] >> (24 - 8 * k)) & 0xffu) << (8 * k + 32);
    const uint32_t m = sub / target;
    return v % (m > 1 ? m : 1u) == 0;
}

// The three signing roots of an item m (wire bytes, Bitvector of sb bytes), 32 bytes each: the selection proof's (SyncAggregatorSelectionData,
// selection domain), the outer signature's (ContributionAndProof, contribution_and_proof domain) and the contribution's (beacon_block_root,
// sync committee domain)
HD void scc_signing_roots(const uint8_t* m, uint32_t sb, const uint8_t* dom_sel, const uint8_t* dom_cap, const uint8_t* dom_sync, uint8_t* sel32,
                          uint8_t* cap32, uint8_t* sync32) {
    uint32_t r[8];
    scc_selection_data_root(m + SCC_SLOT, m + SCC_INDEX, r);
    api_signing_root(r, dom_sel, sel32);
    scc_contribution_and_proof_root(m, sb, r);
    api_signing_root(r, dom_cap, cap32);
    api_chunk_words(m + SCC_ROOT, r);
    api_signing_root(r, dom_sync, sync32);
}

}  // namespace b2

#if defined(__CUDACC__)
#include "syncmsg.cuh"

namespace b2 {

struct scc_args {
    const uint8_t* wire;
    uint64_t wire_len;
    const uint32_t* woff;
    uint32_t n;
    uint32_t size, subnets, sub, sb, sw, ab, target;      // committee_size, subnet_count, subcommittee size, Bitvector bytes and words, aggregate bytes
    uint64_t current_slot, n_val;
    intake_domain dom_sync, dom_sel, dom_cap;
    scm_args M;            // k_scm_index / scm_first_position / k_scm_number: keys, pos_val, size, sub, n_val; the accepted roots' numbering
    // scratch: per item, per hash-table slot, per position, per (root, subnet)
    uint32_t *subnet, *canon, *rslot, *rtab, *bw, *ones;
    uint32_t rtab_mask;
    uint32_t *av_signer, *av_off;
    uint8_t *av_msg, *av_sig;
    uint32_t *members, *item_off;
    uint8_t *fbits, *fmsg, *fsig;
    const uint8_t *av_ok, *fav_ok;
    uint8_t* taken;
    uint32_t* acc;
    unsigned long long* bestkey;
    uint32_t *cnt, *gsrc;
    // outputs
    int32_t* status;
    uint32_t *root_id, *best;
    uint8_t* abits;
    uint32_t* guard;
};

__device__ __forceinline__ const uint8_t* scc_item(const scc_args& A, uint32_t a) { return A.wire + A.woff[a]; }

__global__ void __launch_bounds__(64) k_scc_parse(scc_args A) {
    const uint32_t a = blockIdx.x * blockDim.x + threadIdx.x;
    if (a >= A.n) return;
    const uint32_t begin = A.woff[a], end = A.woff[a + 1];
    const uint8_t* w = A.wire + begin;
    int32_t st = 1;
    uint32_t s = 0, pos = VOTE_NONE, ones = 0;
    uint64_t v = 0;
    if (begin > end || end > A.wire_len) {
        if (A.guard) atomicOr(A.guard, (uint32_t)GUARD_BAD_ROW);
    } else if (end - begin == SCC_FIXED + A.sb && (w[SCC_BITS + A.sb - 1] >> (A.sub & 7) == 0 || (A.sub & 7) == 0)) {
        // the right length and no Bitvector bit past sub
        for (uint32_t k = 0; k < A.sb; k++) ones += __popc((uint32_t)w[SCC_BITS + k]);
        const uint64_t idx = intake_le64(w + SCC_INDEX);
        v = intake_le64(w);
        if (intake_le64(w + SCC_SLOT) != A.current_slot) st = 2;
        else if (idx >= A.subnets) st = 3;
        else if (ones == 0) st = 4;
        else if (!scc_is_aggregator(w + scc_proof(A.sb), A.sub, A.target)) st = 5;
        else if (v >= A.n_val) st = 6;      // n_val < 2^32: v fits a u32 from here on
        else if ((pos = scm_first_position(A.M, (uint32_t)v, (uint32_t)idx)) == VOTE_NONE) st = 7;
        else st = 0;
        s = (uint32_t)idx;
    }
    const bool go = st == 0;
    A.status[a] = st;
    A.subnet[a] = go ? s : VOTE_NONE;
    A.canon[a] = go ? pos : VOTE_NONE;
    A.ones[a] = go ? ones : 0u;
    // the bit row as little-endian words (checks 8 and the aggregate's bits) and as the FastAggregateVerify row
    uint32_t* bw = A.bw + (uint64_t)a * A.sw;
    uint8_t* fb = A.fbits + (uint64_t)a * A.sb;
    for (uint32_t k = 0; k < A.sw; k++) {
        uint32_t x = 0;
        for (uint32_t j = 0; j < 4; j++) {
            const uint32_t b = 4 * k + j;
            if (go && b < A.sb) x |= (uint32_t)w[SCC_BITS + b] << (8 * j);
        }
        bw[k] = x;
    }
    for (uint32_t k = 0; k < A.sb; k++) fb[k] = go ? w[SCC_BITS + k] : 0;
    uint32_t* mrow = A.members + (uint64_t)a * A.sub;
    for (uint32_t i = 0; i < A.sub; i++) mrow[i] = go ? A.M.pos_val[s * A.sub + i] : 0u;
    A.item_off[a] = a * A.sub;
    if (a == A.n - 1) A.item_off[A.n] = A.n * A.sub;
    A.av_off[2 * a] = 2 * a;
    A.av_off[2 * a + 1] = 2 * a + 1;
    if (a == A.n - 1) A.av_off[2 * A.n] = 2 * A.n;
    const uint32_t signer = go ? (uint32_t)v : 0u;
    A.av_signer[2 * a] = signer;
    A.av_signer[2 * a + 1] = signer;
    uint8_t* m0 = A.av_msg + 64 * (uint64_t)a;
    uint8_t* fm = A.fmsg + 32 * (uint64_t)a;
    if (go) {
        scc_signing_roots(w, A.sb, A.dom_sel.b, A.dom_cap.b, A.dom_sync.b, m0, m0 + 32, fm);
    } else {
        for (int k = 0; k < 64; k++) m0[k] = 0;
        for (int k = 0; k < 32; k++) fm[k] = 0;
    }
    uint8_t* sg = A.av_sig + 192 * (uint64_t)a;
    uint8_t* fs = A.fsig + 96 * (uint64_t)a;
    for (int k = 0; k < 96; k++) {
        sg[k] = go ? w[scc_proof(A.sb) + k] : 0;
        sg[96 + k] = go ? w[scc_outer(A.sb) + k] : 0;
        fs[k] = go ? w[scc_sig(A.sb) + k] : 0;
    }
    A.rslot[a] = VOTE_NONE;
    if (!go) return;
    // the root's slot in the insert-only table: items with byte-equal roots meet in one slot
    const uint8_t* r = w + SCC_ROOT;
    uint32_t h = ((uint32_t)r[0] | (uint32_t)r[1] << 8 | (uint32_t)r[2] << 16 | (uint32_t)r[3] << 24) ^ (uint32_t)r[31] << 24;
    h = (h * 0x9e3779b9u) >> 7;
    h &= A.rtab_mask;
    for (;;) {      // the table holds at least 2n slots: a free one is always found
        const uint32_t o = atomicCAS(&A.rtab[h], VOTE_NONE, a);
        if (o == VOTE_NONE) break;
        const uint8_t* e = scc_item(A, o) + SCC_ROOT;
        bool eq = true;
        for (int k = 0; k < 32 && eq; k++) eq = r[k] == e[k];
        if (eq) break;
        h = (h + 1) & A.rtab_mask;
    }
    A.rslot[a] = h;
}

// Warp per subnet: its candidates (status 0 after checks 1-7) in list order.  Check 8 compares the item's root slot and bits with each
// item accepted before on the subnet (at most sub of them: one per aggregator), check 9 reads the accepted flag at the aggregator's first
// position in the subnet; only then do the signature verdicts count.  An accepted item joins acc[s * sub ..].
__global__ void __launch_bounds__(32) k_scc_order(scc_args A) {
    const uint32_t s = blockIdx.x, lane = threadIdx.x;
    uint32_t* acc = A.acc + (uint64_t)s * A.sub;
    uint32_t nacc = 0;
    for (uint32_t c0 = 0; c0 < A.n; c0 += 32) {
        const uint32_t x = c0 + lane;
        unsigned m = __ballot_sync(B2_FULL_MASK, x < A.n && A.subnet[x] == s);
        while (m) {
            const uint32_t a = c0 + __ffs(m) - 1;
            m &= m - 1;
            const uint32_t ra = A.rslot[a];
            const uint32_t* wa = A.bw + (uint64_t)a * A.sw;
            bool shadow = false;      // check 8: an accepted item of the same root whose bits cover this item's
            for (uint32_t k = lane; k < nacc && !shadow; k += 32) {
                const uint32_t b = acc[k];
                if (A.rslot[b] != ra) continue;
                const uint32_t* wb = A.bw + (uint64_t)b * A.sw;
                bool sub = true;
                for (uint32_t q = 0; q < A.sw && sub; q++) sub = (wa[q] & ~wb[q]) == 0;
                shadow = sub;
            }
            shadow = __any_sync(B2_FULL_MASK, shadow);
            const uint32_t p = A.canon[a];
            int32_t st;
            if (shadow) st = 8;
            else if (A.taken[p]) st = 9;
            else if (!A.av_ok[2 * a]) st = 10;
            else if (!A.av_ok[2 * a + 1]) st = 11;
            else if (!A.fav_ok[a]) st = 12;
            else st = 0;
            if (lane == 0) {
                A.status[a] = st;
                if (st == 0) {
                    acc[nacc] = a;
                    A.taken[p] = 1;
                }
            }
            nacc += st == 0;
            __syncwarp();
        }
    }
}

// thread per item: the slot of k_scm_number (VOTE_NONE unless accepted), and the first accepted item of each root slot
__global__ void __launch_bounds__(128) k_scc_claim(scc_args A) {
    const uint32_t a = blockIdx.x * blockDim.x + threadIdx.x;
    if (a >= A.n) return;
    const bool ok = A.status[a] == 0;
    const uint32_t h = ok ? A.rslot[a] : VOTE_NONE;
    A.M.slot_of[a] = h;
    if (ok) atomicMin(&A.M.rmin[h], a);
}

// thread per accepted item: bestkey[root][subnet] = max(ones << 32 | ~a): the most bits, ties to the smaller list index
__global__ void __launch_bounds__(128) k_scc_best(scc_args A) {
    const uint32_t a = blockIdx.x * blockDim.x + threadIdx.x;
    if (a >= A.n || A.status[a] != 0) return;
    atomicMax(&A.bestkey[(uint64_t)A.root_id[a] * A.subnets + A.subnet[a]], (unsigned long long)A.ones[a] << 32 | (uint32_t)~a);
}

// thread per root r < n: best[r][*], the aggregate's bit row (bit s * sub + i = bit i of best[r][s]'s row), and the present subnets (the
// root's segment size).  Roots >= n_roots have no accepted item: none, zero rows, empty segments.
__global__ void __launch_bounds__(128) k_scc_rows(scc_args A) {
    const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= A.n) return;
    uint32_t c = 0;
    for (uint32_t s = 0; s < A.subnets; s++) {
        const unsigned long long k = A.bestkey[(uint64_t)r * A.subnets + s];
        A.best[(uint64_t)r * A.subnets + s] = k ? ~(uint32_t)k : VOTE_NONE;
        c += k != 0;
    }
    A.cnt[r] = c;
    uint8_t* row = A.abits + (uint64_t)r * A.ab;
    for (uint32_t j = 0; j < A.ab; j++) {
        uint32_t x = 0;
        for (uint32_t i = 0; i < 8; i++) {
            const uint32_t q = 8 * j + i, s = q / A.sub, t = q - s * A.sub;
            if (q >= A.size) break;
            const unsigned long long k = A.bestkey[(uint64_t)r * A.subnets + s];
            if (k && (A.bw[(uint64_t)(~(uint32_t)k) * A.sw + (t >> 5)] >> (t & 31) & 1u)) x |= 1u << i;
        }
        row[j] = (uint8_t)x;
    }
}

// thread per root: its best items in subnet order at its segment (cnt now holds the exclusive scan)
__global__ void __launch_bounds__(128) k_scc_gather(scc_args A) {
    const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= A.n) return;
    uint32_t o = A.cnt[r];
    for (uint32_t s = 0; s < A.subnets; s++) {
        const uint32_t b = A.best[(uint64_t)r * A.subnets + s];
        if (b != VOTE_NONE) A.gsrc[o++] = b;
    }
}

}  // namespace b2
#endif
