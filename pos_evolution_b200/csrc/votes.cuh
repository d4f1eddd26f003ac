// votes.cuh -- grouping an epoch's individual signatures by the vote (AttestationData) each member signed, so that the epoch kernels
// aggregate and verify one segment per vote instead of one per committee (pos-evolution.md:714-717, :722-754).  Included by b200pos.cu only.
//
// Committee c holds members [off[c], off[c+1]) and the vote ids [vote_off[c], vote_off[c+1]).  One CTA per committee stable-sorts the
// committee's positions by local vote id (vote[j] - vote_off[c]) with a counting sort; non-attesters (0xFFFFFFFF, or an id outside the
// committee's range) sort last and so fall into the segment of the committee's last vote, with their signature slots replaced by the
// infinity encoding and their bits clear.  Every vote's segment therefore stays inside its committee's range: seg_off[vote_off[c]] ==
// off[c], seg_off[n_votes] == off[n_committees], and no scan crosses committees.
#pragma once
#include <stdint.h>

#include "kernels.cuh"

namespace b2 {

constexpr uint32_t VOTES_THREADS = 256;
constexpr uint32_t VOTES_MAX_MEMBERS = 2048;      // 8 * bits_stride, bits_stride <= 256
constexpr uint32_t VOTE_NONE = 0xffffffffu;

struct vote_group_args {
    const uint32_t *vote, *vote_off, *off, *members;
    uint32_t n_committees, n_votes, bits_stride;
    uint64_t n_sig;
    const uint8_t* sig96;            // signatures of the members [off[c_begin], off[c_end]) only
    uint32_t c_begin, c_end;
    uint8_t* sig96_out;              // the same range, grouped
    uint32_t *members_out, *pos_out, *seg_off, *seg_off_loc;
    uint8_t *bits_out, *agg_bits_out;
    uint32_t* guard;
};

// the first `count` bits of a bit row, byte i
__device__ __forceinline__ uint8_t votes_prefix_byte(uint32_t count, uint32_t i) {
    if (count >= 8 * i + 8) return 0xff;
    return count > 8 * i ? (uint8_t)((1u << (count - 8 * i)) - 1) : 0;
}

__global__ void __launch_bounds__(VOTES_THREADS) k_votes_group(vote_group_args A) {
    __shared__ uint16_t key[VOTES_MAX_MEMBERS];      // local vote id per committee position; ns = not attesting
    __shared__ uint16_t dst[VOTES_MAX_MEMBERS];      // grouped position per committee position
    __shared__ uint32_t start[VOTES_MAX_MEMBERS + 2];      // per local vote: members before it (then the placement cursor)
    __shared__ uint32_t part[VOTES_THREADS];
    const uint32_t c = blockIdx.x, tid = threadIdx.x, bs = A.bits_stride;

    // the whole vote_off array: starts at 0, strictly increasing, ends at n_votes -- or no vote of the epoch is trusted
    uint32_t bad = tid == 0 && (A.vote_off[0] != 0 || A.vote_off[A.n_committees] != A.n_votes);
    for (uint32_t i = tid; i < A.n_committees; i += VOTES_THREADS) bad |= A.vote_off[i] >= A.vote_off[i + 1];
    if (__syncthreads_or((int)bad)) {
        if (c == 0 && tid == 0 && A.guard) atomicOr(A.guard, (uint32_t)GUARD_BAD_ROW);
        // every vote empty: all offsets 0, all bit rows clear (grid-stride over the epoch's entries)
        const uint64_t stride = (uint64_t)gridDim.x * VOTES_THREADS;
        for (uint64_t i = (uint64_t)c * VOTES_THREADS + tid; i <= A.n_votes; i += stride) {
            A.seg_off[i] = 0;
            if (A.seg_off_loc) A.seg_off_loc[i] = 0;
        }
        for (uint64_t i = (uint64_t)c * VOTES_THREADS + tid; i < (uint64_t)A.n_votes * bs; i += stride) A.bits_out[i] = A.agg_bits_out[i] = 0;
        return;
    }

    const uint32_t v0 = A.vote_off[c], nv = A.vote_off[c + 1] - v0;
    const uint32_t o0 = A.off[c], o1 = A.off[c + 1];
    const bool local = c >= A.c_begin && c < A.c_end;
    const uint32_t base = A.off[A.c_begin], lv0 = A.vote_off[A.c_begin];
    // a malformed committee row (reversed, past the signatures, larger than the bit row), more votes than bit positions, or (in this
    // rank's range) a row outside the local signature range: every vote of the committee is empty
    bool row_ok = o0 <= o1 && o1 <= A.n_sig && o1 - o0 <= 8 * bs && nv <= 8 * bs;
    if (local) row_ok = row_ok && o0 >= base && o1 <= A.off[A.c_end];
    const uint32_t m = row_ok ? o1 - o0 : 0;
    const uint32_t safe0 = o0 <= A.n_sig ? o0 : (uint32_t)A.n_sig;
    if (!row_ok && tid == 0 && A.guard) atomicOr(A.guard, (uint32_t)GUARD_BAD_ROW);
    const uint32_t ns = row_ok ? nv : 0;      // buckets 0 .. ns-1 are votes, bucket ns is "not attesting"

    for (uint32_t i = tid; i <= ns + 1; i += VOTES_THREADS) start[i] = 0;
    __syncthreads();
    uint32_t bad_index = 0;
    for (uint32_t j = tid; j < m; j += VOTES_THREADS) {
        const uint32_t v = A.vote[o0 + j];
        uint32_t l = v - v0;      // (wraps for v < v0)
        if (l >= ns) {
            bad_index |= v != VOTE_NONE;
            l = ns;
        }
        key[j] = (uint16_t)l;
        atomicAdd(&start[l + 1], 1u);
    }
    if (__syncthreads_or((int)bad_index) && tid == 0 && A.guard) atomicOr(A.guard, (uint32_t)GUARD_BAD_INDEX);
    // inclusive scan of start[1 .. ns+1]: each thread sums a chunk, the chunk sums are scanned, the chunks add their prefix
    const uint32_t nb = ns + 1, chunk = (nb + VOTES_THREADS - 1) / VOTES_THREADS;
    const uint32_t b0 = 1 + tid * chunk, b1 = min(1 + (tid + 1) * chunk, nb + 1);
    uint32_t sum = 0;
    for (uint32_t i = b0; i < b1; i++) sum += start[i];
    part[tid] = sum;
    __syncthreads();
    for (uint32_t d = 1; d < VOTES_THREADS; d <<= 1) {
        const uint32_t x = tid >= d ? part[tid - d] : 0;
        __syncthreads();
        part[tid] += x;
        __syncthreads();
    }
    uint32_t run = tid ? part[tid - 1] : 0;
    for (uint32_t i = b0; i < b1; i++) {
        run += start[i];
        start[i] = run;
    }
    __syncthreads();

    // per vote: its segment, its prefix bit row, its aggregation_bits row over committee positions
    const uint32_t n_att = start[ns];
    for (uint32_t l = tid; l < nv; l += VOTES_THREADS) {
        const uint32_t s = l < ns ? start[l] : n_att;
        A.seg_off[v0 + l] = row_ok ? o0 + s : safe0;
        if (local && A.seg_off_loc) A.seg_off_loc[v0 + l - lv0] = row_ok ? o0 + s - base : 0;
    }
    if (c == A.n_committees - 1 && tid == 0) A.seg_off[A.n_votes] = row_ok ? o1 : safe0;
    if (local && c == A.c_end - 1 && tid == 0 && A.seg_off_loc) A.seg_off_loc[A.vote_off[A.c_end] - lv0] = row_ok ? o1 - base : 0;
    for (uint64_t i = tid; i < (uint64_t)nv * bs; i += VOTES_THREADS) {
        const uint32_t l = (uint32_t)(i / bs), byte = (uint32_t)(i - (uint64_t)l * bs);
        const uint32_t count = l < ns ? start[l + 1] - start[l] : 0;
        A.bits_out[(uint64_t)(v0 + l) * bs + byte] = votes_prefix_byte(count, byte);
        uint32_t b = 0;
        for (uint32_t k = 0; k < 8; k++) {
            const uint32_t j = 8 * byte + k;
            b |= (j < m && key[j] == l) ? 1u << k : 0u;
        }
        A.agg_bits_out[(uint64_t)(v0 + l) * bs + byte] = (uint8_t)b;
    }
    if (m == 0) return;
    __syncthreads();      // the rows above read start[]; the placement below turns it into cursors

    // stable placement: warp 0 walks the positions in order, 32 at a time; equal keys of one step rank by lane
    if (tid < 32) {
        for (uint32_t j0 = 0; j0 < m; j0 += 32) {
            const uint32_t j = j0 + tid;
            const bool live = j < m;
            const uint32_t k = live ? key[j] : 0xffffu;
            const uint32_t peers = __match_any_sync(0xffffffffu, k);
            const uint32_t rank = __popc(peers & ((1u << tid) - 1));
            const uint32_t at = live ? start[k] : 0;
            __syncwarp();      // every lane has read its cursor before the first lane of each key moves it
            if (live) {
                dst[j] = (uint16_t)(at + rank);
                if (rank == 0) start[k] = at + __popc(peers);
            }
            __syncwarp();
        }
    }
    __syncthreads();

    for (uint32_t j = tid; j < m; j += VOTES_THREADS) {
        const uint32_t p = o0 + dst[j];
        A.members_out[p] = A.members[o0 + j];
        A.pos_out[p] = j;
    }
    if (!local) return;
    // signatures, word by word (coalesced over member x word); a non-attester's slot becomes the infinity encoding 0xc0 || 0^95
    const uint32_t* in = reinterpret_cast<const uint32_t*>(A.sig96) + (uint64_t)(o0 - base) * 24;
    uint32_t* out = reinterpret_cast<uint32_t*>(A.sig96_out) + (uint64_t)(o0 - base) * 24;
    for (uint32_t i = tid; i < m * 24; i += VOTES_THREADS) {
        const uint32_t j = i / 24, w = i - j * 24;
        out[(uint64_t)dst[j] * 24 + w] = key[j] < ns ? in[i] : (w == 0 ? 0xc0u : 0u);
    }
}

// A vote nobody attested reads like an empty segment of b2_epoch_dev: aggregate status 2 and 96 zero bytes (its verdict is 0 already:
// no pubkey is selected).  The last vote of a committee without attesters holds the committee's infinity slots, so its segment is
// not empty; this makes it so.  Bit 0 of a grouped row is set exactly when the vote has an attester.
__global__ void k_votes_empty(const uint8_t* __restrict__ bits, uint32_t bits_stride, uint32_t n_votes, uint8_t* agg_sig96, int32_t* agg_status) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (uint64_t)n_votes * 24) return;
    const uint32_t v = (uint32_t)(i / 24), w = (uint32_t)(i - (uint64_t)v * 24);
    if (bits[(uint64_t)v * bits_stride] & 1) return;
    uint8_t* o = agg_sig96 + 96 * (uint64_t)v + 4 * w;
    o[0] = o[1] = o[2] = o[3] = 0;
    if (w == 0 && agg_status) agg_status[v] = 2;
}

}  // namespace b2
