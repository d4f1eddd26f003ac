// blockatt_electra.cuh -- process_attestation for the Electra (EIP-7549) on-chain Attestation with Deneb's (EIP-7045) inclusion window
// (upstream consensus-specs, Deneb and Electra beacon-chain.md), for the attestations of a run of blocks of one chain in one epoch e,
// block-atomic as b2_block_attestations is (blockatt.cuh).  One aggregate names up to MAX_COMMITTEES_PER_SLOT committees of one slot in
// committee_bits, and its aggregation_bits are their bit rows back to back.  The decode and checks are __host__ __device__ so that
// tests/hostsim can run them on the CPU; the kernels are for nvcc only.  Included by b200pos.cu only.
//
//   k_bae_parse     warp per attestation: its block, the container (bae_decode), checks 1-12 against the block's slot (bae_check, the
//                   committee loop's bit scans spread over the warp), the Deneb flag mask, the signature, data and attester domain
//   k_bae_rows      CTA per attestation: the member row (its committees' members back to back) and the bit row (the Bitlist without its
//                   delimiter), both zero padded to R = BAE_CHUNK * ceil(row_max / BAE_CHUNK) members; the chunk offsets of the split sum
//   k_signing_roots (kernels.cuh) thread per attestation
//   FastAggregateVerify with the split key sum: k_g1_gather_tma<false> (gather.cuh, unchanged) with one warp per BAE_CHUNK members of a
//   row, each chunk taken as an aggregate of its own, then k_bae_pk_combine (warp per attestation) adds the partial sums with the
//   complete Jacobian addition into the aggregate keys verify_main pairs
//   k_ba_blocks, k_part_phase1-3, k_ba_rewards (blockatt.cuh, kernels.cuh) as for phase 0, over the padded rows; a failed
//                   FastAggregateVerify is status 13
//
// Wire form: offset u32 | data 128 | signature 96 | committee_bits ceil(M / 8) | aggregation_bits Bitlist, M = max_committees_per_slot.
#pragma once
#include "platform.cuh"

namespace b2 {

constexpr uint32_t BAE_DATA = 4, BAE_SIG = 132, BAE_CBITS = 228;
// Members per chunk of the split key sum: one warp of k_g1_gather_tma each.  A multiple of 512 (the gather's staging unit), so a chunk's
// bit row starts on a 64-byte boundary.  Chosen by measurement (DESIGN.md section 6): at 256 aggregates of 32 768 members the key sum takes
// the least time at 2 048 and 4 096, and at 8 aggregates 2 048 still finishes well inside the hash-to-G2 it runs beside.
constexpr uint32_t BAE_CHUNK = 2048;

HD uint32_t bae_fixed(uint32_t M) { return BAE_CBITS + (M + 7) / 8; }
HD uint64_t bae_le64(const uint8_t* p) {
    uint64_t v = 0;
    for (int i = 7; i >= 0; i--) v = v << 8 | p[i];
    return v;
}

// checks 1-3 of the container w[0, len): 0 and the Bitlist's length in bits, or 1 (truncated, offset != fixed size, a committee_bits padding
// bit set), 2 (no Bitlist byte, or no delimiter bit), 3 (more than `limit` bits)
HD int32_t bae_decode(const uint8_t* w, uint64_t len, uint32_t M, uint64_t limit, uint32_t& nbits) {
    const uint32_t F = bae_fixed(M);
    nbits = 0;
    if (len < F || ((uint32_t)w[0] | (uint32_t)w[1] << 8 | (uint32_t)w[2] << 16 | (uint32_t)w[3] << 24) != F) return 1;
    if ((M & 7) && (w[F - 1] >> (M & 7)) != 0) return 1;
    if (len == F || w[len - 1] == 0) return 2;
    uint32_t top = 7;
    while (!((w[len - 1] >> top) & 1)) top--;
    const uint64_t n = 8 * (len - F - 1) + top;
    if (n > limit) return 3;
    nbits = (uint32_t)n;
    return 0;
}

// whether a bit of bl in [lo, hi) is set, over the bytes lane, lane + nl, ... of that range (the caller ORs the lanes)
HD bool bae_any_bit(const uint8_t* bl, uint32_t lo, uint32_t hi, uint32_t lane, uint32_t nl) {
    bool any = false;
    if (lo >= hi) return false;
    for (uint32_t k = (lo >> 3) + lane; k <= ((hi - 1) >> 3); k += nl) {
        uint32_t x = bl[k];
        if (8 * k < lo) x &= 0xffu << (lo & 7);
        if (8 * k + 8 > hi) x &= (1u << (hi - 8 * k)) - 1u;
        any |= x != 0;
    }
    return any;
}

struct bae_in {
    const uint8_t* w;                          // the container, len bytes
    uint64_t len, bslot, e;                    // the including block's slot, e = its epoch
    const uint32_t* off;                       // committee layout (b2_block_attestations'), n_sig member slots
    uint64_t n_sig;
    uint32_t M, max_vpc, cps_prev, cps_cur, spe, min_delay, isqrt_spe, row_max;
    const uint8_t* chain_roots;                // u8[2 * spe][32]: slot s at s + spe - start(e)
    const uint8_t* justified80;                // previous_justified_checkpoint, then current_justified_checkpoint
};
struct bae_out {
    uint32_t nbits, c0;                        // the Bitlist's length; committee (target epoch, data.slot, 0)
    unsigned long long cmask;                  // committee_bits
    uint32_t mask;                             // participation flags; 0 unless checks 1-11 pass
    bool cur, bad_row;                         // target is e; a malformed committee row was met
};

// checks 1-12 of one attestation; `any(x)` ORs x over the nl callers that run this with lanes 0 .. nl - 1 (identity when nl == 1)
template <class Any>
HD int32_t bae_check(const bae_in& I, uint32_t lane, uint32_t nl, Any any, bae_out& O) {
    O = bae_out{};
    const uint64_t limit = (uint64_t)I.max_vpc * I.M;
    int32_t st = bae_decode(I.w, I.len, I.M, limit, O.nbits);
    if (st) return st;
    const uint8_t* d = I.w + BAE_DATA;
    const uint8_t* cb = I.w + BAE_CBITS;
    const uint8_t* bl = I.w + bae_fixed(I.M);
    const uint64_t slot = bae_le64(d), index = bae_le64(d + 8), tgt = bae_le64(d + 88), spe = I.spe, e = I.e;
    O.cur = tgt == e;
    if (!O.cur && (e == 0 || tgt != e - 1)) return 4;
    if (tgt != slot / spe) return 5;
    if (slot + I.min_delay > I.bslot) return 6;      // Deneb: no upper bound
    if (index != 0) return 7;
    const uint32_t cps = O.cur ? I.cps_cur : I.cps_prev;
    // slot - start(tgt) < spe by check 5
    O.c0 = (O.cur ? I.cps_prev * I.spe : 0u) + (uint32_t)(slot - tgt * spe) * cps;
    uint32_t coff = 0;
    for (uint32_t ci = 0; ci < I.M; ci++) {
        if (!((cb[ci >> 3] >> (ci & 7)) & 1)) continue;
        if (ci >= cps) return 8;
        const uint32_t o0 = I.off[O.c0 + ci], o1 = I.off[O.c0 + ci + 1];
        if (!(o0 <= o1 && o1 <= I.n_sig && o1 - o0 <= I.row_max - coff)) {
            O.bad_row = true;                  // a malformed row matches no Bitlist
            return 10;
        }
        if ((uint64_t)coff + (o1 - o0) > O.nbits) return 10;
        if (!any(bae_any_bit(bl, coff, coff + (o1 - o0), lane, nl))) return 9;
        coff += o1 - o0;
        O.cmask |= 1ull << ci;
    }
    if (coff != O.nbits) return 10;
    const uint8_t* J = I.justified80 + (O.cur ? 40 : 0);
    for (int k = 0; k < 40; k++)
        if (d[48 + k] != J[k]) return 11;
    // get_block_root(target epoch) = the root at start(tgt); get_block_root_at_slot(data.slot); slot >= start(e - 1) by check 5
    const uint8_t* troot = I.chain_roots + 32ull * (O.cur ? spe : 0u);
    const uint8_t* hroot = I.chain_roots + 32ull * (slot + spe - e * spe);
    bool target = true, head = true;
    for (int k = 0; k < 32; k++) {
        target &= d[96 + k] == troot[k];
        head &= d[16 + k] == hroot[k];
    }
    const uint64_t delay = I.bslot - slot;
    O.mask = (delay <= I.isqrt_spe ? 1u : 0u) | (target ? 2u : 0u) | (target && head && delay == I.min_delay ? 4u : 0u);
    return O.cmask ? 0 : 12;
}

}  // namespace b2

#if defined(__CUDACC__)
#include "blockatt.cuh"

namespace b2 {

struct bae_args {
    ba_args B;                                 // block rows, statuses, accept masks, numerators, FastAggregateVerify rows (R-member rows)
    uint32_t M, max_vpc, row_max, R, n_chunks; // R = n_chunks * BAE_CHUNK, the padded row
    uint64_t n_sig;
    const uint32_t* off;
    // per attestation: the Bitlist's length, committee_bits and the first committee, written by k_bae_parse for k_bae_rows
    uint32_t *nbits, *c0;
    unsigned long long* cmask;
    uint32_t* chunk_off;                       // u32[n * n_chunks + 1]: chunk v = members [v * BAE_CHUNK, (v + 1) * BAE_CHUNK)
};

struct bae_warp_any {
    __device__ bool operator()(bool x) const { return __any_sync(B2_FULL_MASK, x); }
};

__global__ void __launch_bounds__(128) k_bae_parse(bae_args A) {
    const ba_args& B = A.B;
    const uint32_t a = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (a >= B.n) return;
    const uint32_t b = ba_block_of(B, a);
    const uint32_t begin = B.woff[a], end = B.woff[a + 1];
    const uint8_t* w = B.wire + begin;
    int32_t st = 1;
    bae_out O = {};
    if (b != VOTE_NONE && begin <= end && end <= B.wire_len) {
        const uint64_t bslot = B.block_slot[b];
        const bae_in I = {w, end - begin, bslot, B.block_slot[0] / B.slots_per_epoch, A.off, A.n_sig, A.M, A.max_vpc, B.cps_prev, B.cps_cur,
                          B.slots_per_epoch, B.min_delay, B.isqrt_spe, A.row_max, B.chain_roots, B.justified.b};
        st = bae_check(I, lane, 32, bae_warp_any{}, O);
        if (O.bad_row && lane == 0 && B.guard) atomicOr(B.guard, (uint32_t)GUARD_BAD_ROW);
    } else if (lane == 0 && B.guard) {
        atomicOr(B.guard, (uint32_t)GUARD_BAD_ROW);
    }
    // what FastAggregateVerify reads (all zero unless the attestation passed checks 1-12)
    const bool go = st == 0;
    for (uint32_t k = lane; k < 96; k += 32) B.sig96[96 * (uint64_t)a + k] = go ? w[BAE_SIG + k] : 0;
    for (uint32_t k = lane; k < 128; k += 32) B.data128[128 * (uint64_t)a + k] = go ? w[BAE_DATA + k] : 0;
    B.dom32[32 * (uint64_t)a + lane] = go ? B.dom[O.cur].b[lane] : 0;
    if (lane == 0) {
        B.status[a] = st;
        B.flag_mask[a] = (uint8_t)O.mask;
        B.blk_of[a] = b;
        B.cur[a] = O.cur;
        A.nbits[a] = go ? O.nbits : 0u;
        A.c0[a] = O.c0;
        A.cmask[a] = go ? O.cmask : 0ull;
    }
}

// CTA per attestation: member row and bit row of R members (zero past the Bitlist), the row offsets k_part_phase1-3 read and the chunk
// offsets of the split key sum
__global__ void __launch_bounds__(256) k_bae_rows(bae_args A) {
    const ba_args& B = A.B;
    const uint32_t a = blockIdx.x, t = threadIdx.x;
    if (a >= B.n) return;
    const uint32_t nbits = A.nbits[a], R = A.R;
    const uint8_t* bl = B.wire + B.woff[a] + bae_fixed(A.M);
    uint8_t* brow = B.bits + (uint64_t)a * (R / 8);
    for (uint32_t k = t; k < R / 8; k += blockDim.x) {
        uint32_t x = 0;
        if (8 * k < nbits) {
            x = bl[k];
            if (8 * k + 8 > nbits) x &= (1u << (nbits & 7u)) - 1u;
        }
        brow[k] = (uint8_t)x;
    }
    uint32_t* mrow = B.members_out + (uint64_t)a * R;
    uint32_t coff = 0;
    unsigned long long m = A.cmask[a];
    while (m) {
        const uint32_t c = A.c0[a] + (uint32_t)__ffsll((long long)m) - 1;
        m &= m - 1;
        const uint32_t o0 = A.off[c], size = A.off[c + 1] - o0;      // checked by k_bae_parse
        for (uint32_t j = t; j < size; j += blockDim.x) mrow[coff + j] = B.members[o0 + j];
        coff += size;
    }
    for (uint32_t j = coff + t; j < R; j += blockDim.x) mrow[j] = 0u;
    for (uint32_t k = t; k < A.n_chunks; k += blockDim.x) A.chunk_off[a * A.n_chunks + k] = (a * A.n_chunks + k) * BAE_CHUNK;
    if (t == 0) {
        B.item_off[a] = a * R;
        if (a == B.n - 1) {
            B.item_off[B.n] = B.n * R;
            A.chunk_off[B.n * A.n_chunks] = B.n * R;
        }
    }
}

// warp per attestation: the sum of its n_chunks partial keys (complete Jacobian additions: a partial sum may be infinity, equal to another or
// its negative) and the OR of their failure bits; empty when every chunk was
__global__ void __launch_bounds__(128) k_bae_pk_combine(const uint32_t* __restrict__ part_jac, const uint8_t* __restrict__ part_st, uint32_t n_chunks,
                                                        uint32_t n, uint32_t* out_jac, uint8_t* out_status) {
    const uint32_t a = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (a >= n) return;
    g1_jac acc = pt_inf<fp>();
    uint32_t status = 0, cnt = 0;
#pragma unroll 1
    for (uint32_t k = lane; k < n_chunks; k += 32) {
        const uint64_t v = (uint64_t)a * n_chunks + k;
        const uint32_t s = part_st[v];
        status |= s & (PK_INVALID_KEY | PK_BAD_INDEX);
        if (!(s & PK_EMPTY)) cnt++;
        acc = pt_add(acc, load_g1_jac(part_jac + 36 * v));
    }
#pragma unroll 1
    for (int delta = 16; delta >= 1; delta >>= 1) {
        g1_jac other = shfl_down_pod(acc, delta);
        if (lane < (uint32_t)delta) acc = pt_add(acc, other);
    }
    status = __reduce_or_sync(B2_FULL_MASK, status);
    cnt = __reduce_add_sync(B2_FULL_MASK, cnt);
    if (lane == 0) core_g1_finish(acc, status, cnt, a, out_jac, out_status);
}

}  // namespace b2
#endif
