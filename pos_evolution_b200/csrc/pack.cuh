// pack.cuh -- block packing: the proposing-side counterpart of process_attestation (pos-evolution.md:639, :659, :722-754).  Turns a pool
// of aggregates into the block's attestation list: fold disjoint aggregates of one vote, then a weighted max-cover greedy whose value is
// the proposer-reward numerator k_part_phase1..3 credit.  Included by b200pos.cu only.
//
// Why per committee is exact: committees of one participation table are disjoint, so a pick changes only the gains of folded aggregates
// of its own committee; inside a committee the weighted-coverage greedy picks non-increasing gains (submodularity).  The global greedy
// (largest gain, then lowest committee, then lowest folded number) is therefore the merge, by (gain desc, committee asc, step asc), of
// independent per-committee greedy sequences cut at max_out -- one CTA per committee, then one selection.
//
// Stages (b2_pack_attestations_dev):
//   k_g2_decompress       every candidate signature once (undecodable ones are excluded)
//   k_pack_claim          CTA per committee: one atomicOr per member into a per-table validator bitmap -> overlap / repeat = bad pool
//   k_pack_prep           thread per candidate: status, data-id consistency (committee and mask), valid candidates per committee
//   k_pack_scan           exclusive scan of those counts: committee k owns slots off[k] .. off[k+1]
//   k_pack_scatter        candidates into their committee's slots (unordered)
//   k_pack_committee      CTA per committee: pool order (bitonic sort), fold (first fit), greedy; entries (gain, folded slot) at off[k] + step
//   k_pack_select         one CTA: radix select of the max_out-th largest gain, ties cut in (committee, step) order = slot order
//   k_pack_rank           selected entries into pick order
//   k_pack_offsets        constituent offsets of the outputs (CSR) and n_out
//   k_pack_emit           CTA per output: committee, data id, union row, numerator, constituents in pool order
//   k_pack_gather + k_g2_segment_sum + k_g2_finish + k_pack_single   bls.Aggregate of the constituents (one constituent: its own bytes)
#pragma once
#include <stdint.h>

#include "kernels.cuh"

namespace b2 {

constexpr uint32_t PACK_NONE = 0xffffffffu;
constexpr uint32_t PACK_MAX_WORDS = 64;                        // bit rows up to 2048 members (MAX_VALIDATORS_PER_COMMITTEE)
constexpr uint32_t PACK_SMEM_ROWS = 64 * 1024;                 // dynamic shared memory of k_pack_committee: the folded union rows
enum PackStatus : uint8_t { PACK_OK = 0, PACK_UNDECODABLE = 1, PACK_BAD_COMMITTEE = 2 };

struct pack_view {
    const uint32_t *members, *coff;          // committees: members[coff[k] .. coff[k+1])
    const uint8_t* ctable;                   // participation table of committee k (0 current, 1 previous)
    const uint32_t *cand_comm, *cand_data;
    const uint8_t *cand_mask, *bits;
    const uint8_t* dec_st;                   // k_g2_decompress status per candidate
    const uint64_t* eff;
    const uint8_t* part[2];                  // may be null: a table never loaded counts as all-zero
    uint32_t n_comm, n_cand, stride, wstride, max_out;
    uint64_t n_val;
    unsigned long long inc, per_inc;
    // scratch (slot s = off[k] + i belongs to committee k)
    uint32_t *cnt, *off, *list, *fold_of;    // per committee: count / fill cursor, slot offsets; per slot: candidate, its folded slot
    uint32_t *fdata, *fcnt, *frow;           // per folded slot: data id, constituents, union row (wstride words)
    uint8_t* fmask;
    unsigned long long* egain;               // per slot: gain of the committee's step (slot - off[k]); 0 = no entry
    uint32_t* eslot;                         // ... and the folded slot it picked
    uint32_t *claim, *dcomm, *dmask;         // validator bitmaps (one per table); committee and mask per data id
    uint32_t *ctl, *sel, *ord;               // ctl[0] bad pool, ctl[1] selected count; selected slots in slot order, in pick order
    uint8_t* cand_status;
    uint32_t* guard;
};

__device__ __forceinline__ void pack_bad_pool(const pack_view& P) {
    P.ctl[0] = 1;
    if (P.guard) atomicOr(P.guard, (uint32_t)GUARD_BAD_POOL);
}

// PARTICIPATION_FLAG_WEIGHTS (14, 26, 14) summed over the flags of `need`
__device__ __forceinline__ unsigned long long pack_weight(uint32_t need) {
    return 14ull * (need & 1u) + 26ull * ((need >> 1) & 1u) + 14ull * ((need >> 2) & 1u);
}

// word w of a bit row (little-endian bytes, SSZ order), bytes past `stride` and bits at or past `size` cleared
__device__ __forceinline__ uint32_t pack_row_word(const uint8_t* row, uint32_t stride, uint32_t w, uint32_t size) {
    uint32_t x = 0;
#pragma unroll
    for (int b = 0; b < 4; b++)
        if (4 * w + b < stride) x |= (uint32_t)row[4 * w + b] << (8 * b);
    const uint32_t lo = 32 * w;
    if (lo + 32 > size) x &= size > lo ? (1u << (size - lo)) - 1u : 0u;
    return x;
}

// Exclusive block-wide prefix sum of one value per thread; *total = the block's sum.  Every thread must call it.
__device__ __forceinline__ uint32_t pack_block_scan(uint32_t x, uint32_t* s_warp, uint32_t* total) {
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarp = blockDim.x >> 5;
    uint32_t inc = x;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const uint32_t y = __shfl_up_sync(B2_FULL_MASK, inc, d);
        if (lane >= (uint32_t)d) inc += y;
    }
    if (lane == 31) s_warp[warp] = inc;
    __syncthreads();
    uint32_t base = 0, sum = 0;
    for (uint32_t w = 0; w < nwarp; w++) {
        if (w < warp) base += s_warp[w];
        sum += s_warp[w];
    }
    __syncthreads();
    *total = sum;
    return base + inc - x;
}

// Ascending sort of a[0..n) by one CTA (global or shared memory): the bitonic network whose comparators all put the smaller value at the
// lower index (flip stage, then half cleaners), so positions past n act as +infinity and are never touched.
__device__ void pack_block_sort(uint32_t* a, uint32_t n) {
    uint32_t p2 = 1;
    while (p2 < n) p2 <<= 1;
    for (uint32_t k = 2; k <= p2; k <<= 1) {
        for (uint32_t j = k >> 1; j > 0; j >>= 1) {
            for (uint32_t i = threadIdx.x; i < p2 / 2; i += blockDim.x) {
                uint32_t lo, hi;
                if (j == k >> 1) {
                    lo = (i / j) * k + i % j;
                    hi = (i / j) * k + k - 1 - i % j;
                } else {
                    lo = (i / j) * 2 * j + i % j;
                    hi = lo + j;
                }
                if (hi < n) {
                    const uint32_t x = a[lo], y = a[hi];
                    if (x > y) {
                        a[lo] = y;
                        a[hi] = x;
                    }
                }
            }
            __syncthreads();
        }
    }
}

// CTA per committee: claim every member in its table's bitmap; a member claimed twice (overlap inside a table, or a repeat) is a bad
// pool, as are a malformed row and a table byte other than 0 / 1.  A member index >= n_val is skipped (GUARD_BAD_INDEX).
__global__ void __launch_bounds__(128) k_pack_claim(pack_view P) {
    const uint32_t k = blockIdx.x;
    const uint32_t o0 = P.coff[k], o1 = P.coff[k + 1], t = P.ctable[k];
    if (o1 < o0 || o1 - o0 > P.stride * 8u || t > 1) {
        if (threadIdx.x == 0) {
            if (P.guard && t <= 1) atomicOr(P.guard, (uint32_t)GUARD_BAD_ROW);
            pack_bad_pool(P);
        }
        return;
    }
    uint32_t* bm = P.claim + (size_t)t * ((P.n_val + 31) / 32);
    for (uint32_t i = o0 + threadIdx.x; i < o1; i += blockDim.x) {
        const uint32_t v = P.members[i];
        if (v >= P.n_val) {
            if (P.guard) atomicOr(P.guard, (uint32_t)GUARD_BAD_INDEX);
            continue;
        }
        const uint32_t bit = 1u << (v & 31);
        if (atomicOr(&bm[v >> 5], bit) & bit) pack_bad_pool(P);
    }
}

// thread per candidate: status byte, data-id consistency, count of the committee's valid candidates
__global__ void __launch_bounds__(128) k_pack_prep(pack_view P) {
    const uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= P.n_cand) return;
    const uint32_t k = P.cand_comm[c];
    if (k >= P.n_comm) {
        P.cand_status[c] = PACK_BAD_COMMITTEE;
        if (P.guard) atomicOr(P.guard, (uint32_t)GUARD_BAD_INDEX);
        return;
    }
    const uint32_t d = P.cand_data[c], m = P.cand_mask[c] & 7u;
    if (d >= P.n_cand) {
        pack_bad_pool(P);
    } else {
        const uint32_t k0 = atomicCAS(&P.dcomm[d], PACK_NONE, k), m0 = atomicCAS(&P.dmask[d], PACK_NONE, m);
        if ((k0 != PACK_NONE && k0 != k) || (m0 != PACK_NONE && m0 != m)) pack_bad_pool(P);
    }
    const bool ok = P.dec_st[c] != DEC_BAD;
    P.cand_status[c] = ok ? PACK_OK : PACK_UNDECODABLE;
    if (ok) atomicAdd(&P.cnt[k], 1u);
}

// one CTA: off[k] = sum of the counts of committees < k; the counts become fill cursors
__global__ void __launch_bounds__(1024) k_pack_scan(pack_view P) {
    __shared__ uint32_t s_warp[32];
    uint32_t carry = 0;
    for (uint32_t b = 0; b < P.n_comm; b += blockDim.x) {
        const uint32_t k = b + threadIdx.x;
        const uint32_t x = k < P.n_comm ? P.cnt[k] : 0;
        uint32_t total;
        const uint32_t ex = pack_block_scan(x, s_warp, &total);
        if (k < P.n_comm) {
            P.off[k] = carry + ex;
            P.cnt[k] = 0;
        }
        carry += total;
    }
    if (threadIdx.x == 0) P.off[P.n_comm] = carry;
}

__global__ void __launch_bounds__(128) k_pack_scatter(pack_view P) {
    const uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= P.n_cand || P.cand_status[c] != PACK_OK) return;
    const uint32_t k = P.cand_comm[c];
    P.list[P.off[k] + atomicAdd(&P.cnt[k], 1u)] = c;
}

// CTA per committee.  The members' reward units and participation bytes live in shared memory, and so do the folded union rows when
// the committee's candidates fit PACK_SMEM_ROWS (otherwise the rows stay in the global slots, any number of candidates).  A candidate's
// own row is read once, by the fold.
__global__ void __launch_bounds__(256) k_pack_committee(pack_view P) {
    extern __shared__ uint32_t s_rows[];
    __shared__ unsigned long long s_unit[PACK_MAX_WORDS * 32];
    __shared__ uint8_t s_part[PACK_MAX_WORDS * 32];
    __shared__ uint32_t s_crow[PACK_MAX_WORDS];
    __shared__ unsigned long long s_gain[8];
    __shared__ uint32_t s_f[8];
    __shared__ uint32_t s_fit, s_nf, s_pick;
    __shared__ unsigned long long s_pick_gain;
    const uint32_t k = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nwarp = blockDim.x >> 5;
    const uint32_t b0 = P.off[k], n = P.off[k + 1] - b0;
    if (n == 0) return;
    uint32_t* L = P.list + b0;
    pack_block_sort(L, n);                               // pool order (the scatter left them in arrival order)

    const uint32_t o0 = P.coff[k], o1 = P.coff[k + 1];
    const uint32_t size = (o1 >= o0 && o1 - o0 <= P.stride * 8u) ? o1 - o0 : 0;     // a malformed row is a bad pool already
    const uint32_t W = (size + 31) / 32;
    const uint8_t* part = P.part[P.ctable[k] & 1u];
    for (uint32_t j = tid; j < size; j += blockDim.x) {
        const uint32_t v = P.members[o0 + j];
        const bool in = v < P.n_val;
        s_unit[j] = in ? (P.eff[v] / P.inc) * P.per_inc : 0ull;
        s_part[j] = in ? (part ? part[v] : 0) : 7;       // an index outside the registry earns nothing
    }
    const bool smem = (size_t)n * W * 4 <= PACK_SMEM_ROWS;
    const uint32_t rs = smem ? W : P.wstride;            // words per union row
    uint32_t* U = smem ? s_rows : P.frow + (size_t)b0 * P.wstride;
    if (tid == 0) s_nf = 0;

    // fold, first fit per data id, in pool order
    for (uint32_t i = 0; i < n; i++) {
        const uint32_t c = L[i], d = P.cand_data[c];
        for (uint32_t w = tid; w < rs; w += blockDim.x) s_crow[w] = w < W ? pack_row_word(P.bits + (size_t)c * P.stride, P.stride, w, size) : 0u;
        if (tid == 0) s_fit = PACK_NONE;
        __syncthreads();
        const uint32_t nf = s_nf;
        for (uint32_t f = warp; f < nf; f += nwarp) {
            if (P.fdata[b0 + f] != d) continue;
            bool clash = false;
            for (uint32_t w = lane; w < W; w += 32) clash |= (U[(size_t)f * rs + w] & s_crow[w]) != 0;
            if (!__any_sync(B2_FULL_MASK, clash)) {      // the warp's lowest fitting folded aggregate
                if (lane == 0) atomicMin(&s_fit, f);
                break;
            }
        }
        __syncthreads();
        const uint32_t g = s_fit == PACK_NONE ? nf : s_fit;
        for (uint32_t w = tid; w < rs; w += blockDim.x) U[(size_t)g * rs + w] = (g == nf ? 0u : U[(size_t)g * rs + w]) | s_crow[w];
        if (tid == 0) {
            P.fold_of[b0 + i] = b0 + g;
            if (g == nf) {
                P.fdata[b0 + g] = d;
                P.fmask[b0 + g] = P.cand_mask[c] & 7u;
                P.fcnt[b0 + g] = 1;
                s_nf = nf + 1;
            } else {
                P.fcnt[b0 + g] += 1;
            }
        }
        __syncthreads();
    }

    // greedy: up to min(max_out, folded) picks, each the largest gain (lowest folded number on a tie), stopping at gain 0
    const uint32_t nf = s_nf, steps = min(P.max_out, nf);
    uint32_t step = 0;
    for (; step < steps; step++) {
        unsigned long long best = 0;
        uint32_t bf = PACK_NONE;
        for (uint32_t f = warp; f < nf; f += nwarp) {
            const uint32_t m = P.fmask[b0 + f];
            unsigned long long gsum = 0;
            for (uint32_t w = lane; w < W; w += 32) {
                uint32_t x = U[(size_t)f * rs + w];
                while (x) {
                    const uint32_t j = 32 * w + __ffs(x) - 1;
                    x &= x - 1;
                    gsum += s_unit[j] * pack_weight(m & ~(uint32_t)s_part[j]);
                }
            }
#pragma unroll
            for (int dd = 16; dd >= 1; dd >>= 1) gsum += __shfl_xor_sync(B2_FULL_MASK, gsum, dd);
            if (gsum > best) {                            // f rises: a tie keeps the lower folded number
                best = gsum;
                bf = f;
            }
        }
        if (lane == 0) {
            s_gain[warp] = best;
            s_f[warp] = bf;
        }
        __syncthreads();
        if (tid == 0) {
            unsigned long long bg = 0;
            uint32_t pf = PACK_NONE;
            for (uint32_t w = 0; w < nwarp; w++)
                if (s_gain[w] > bg || (s_gain[w] == bg && bg > 0 && s_f[w] < pf)) {
                    bg = s_gain[w];
                    pf = s_f[w];
                }
            s_pick_gain = bg;
            s_pick = pf;
            if (bg > 0) {
                P.egain[b0 + step] = bg;
                P.eslot[b0 + step] = b0 + pf;
            }
        }
        __syncthreads();
        if (s_pick_gain == 0) break;
        const uint32_t f = s_pick, m = P.fmask[b0 + f];
        for (uint32_t w = tid; w < W; w += blockDim.x) {
            uint32_t x = U[(size_t)f * rs + w];
            while (x) {
                const uint32_t j = 32 * w + __ffs(x) - 1;
                x &= x - 1;
                s_part[j] |= (uint8_t)m;
            }
        }
        __syncthreads();
    }
    for (uint32_t p = step + tid; p < n; p += blockDim.x) P.egain[b0 + p] = 0;
    if (smem)                                            // the emit stage reads the union rows from the global slots
        for (uint32_t idx = tid; idx < nf * P.wstride; idx += blockDim.x) {
            const uint32_t f = idx / P.wstride, w = idx % P.wstride;
            P.frow[(size_t)(b0 + f) * P.wstride + w] = w < W ? s_rows[(size_t)f * W + w] : 0u;
        }
}

// One CTA over the entry slots.  T = the max_out-th largest gain (radix select, 8 digits of 8 bits); the selection is every entry with
// gain > T plus the first `need` entries with gain == T in slot order, which is (committee, step) order.  A bad pool selects nothing.
__global__ void __launch_bounds__(1024) k_pack_select(pack_view P) {
    __shared__ uint32_t s_hist[256], s_warp[32];
    __shared__ unsigned long long s_prefix;
    __shared__ uint32_t s_need;
    const uint32_t nv = P.off[P.n_comm];
    uint32_t total = 0;
    for (uint32_t b = 0; b < nv; b += blockDim.x) {
        const uint32_t p = b + threadIdx.x;
        total += __syncthreads_count(p < nv && P.egain[p] != 0);
    }
    if (P.ctl[0]) {
        if (threadIdx.x == 0) P.ctl[1] = 0;
        return;
    }
    unsigned long long T = 0;
    uint32_t need = 0;
    if (total > P.max_out) {
        unsigned long long pmask = 0;
        if (threadIdx.x == 0) {
            s_prefix = 0;
            s_need = P.max_out;
        }
        for (int shift = 56; shift >= 0; shift -= 8) {
            for (uint32_t i = threadIdx.x; i < 256; i += blockDim.x) s_hist[i] = 0;
            __syncthreads();
            const unsigned long long prefix = s_prefix;
            for (uint32_t p = threadIdx.x; p < nv; p += blockDim.x) {
                const unsigned long long g = P.egain[p];
                if (g != 0 && (g & pmask) == prefix) atomicAdd(&s_hist[(g >> shift) & 255u], 1u);
            }
            __syncthreads();
            if (threadIdx.x == 0) {
                uint32_t cum = 0;
                for (int b = 255; b >= 0; b--) {
                    if (cum + s_hist[b] >= s_need) {
                        s_prefix = prefix | ((unsigned long long)b << shift);
                        s_need -= cum;
                        break;
                    }
                    cum += s_hist[b];
                }
            }
            pmask |= 255ull << shift;
            __syncthreads();
        }
        T = s_prefix;
        need = s_need;
    }
    uint32_t carry_eq = 0, carry_sel = 0;
    for (uint32_t b = 0; b < nv; b += blockDim.x) {
        const uint32_t p = b + threadIdx.x;
        const unsigned long long g = p < nv ? P.egain[p] : 0ull;
        const bool gt = g != 0 && g > T, eq = g != 0 && g == T;
        uint32_t n_eq, n_sel;
        const uint32_t eq_rank = carry_eq + pack_block_scan(eq ? 1u : 0u, s_warp, &n_eq);
        const bool take = gt || (eq && eq_rank < need);
        const uint32_t pos = carry_sel + pack_block_scan(take ? 1u : 0u, s_warp, &n_sel);
        if (take) P.sel[pos] = p;
        carry_eq += n_eq;
        carry_sel += n_sel;
    }
    if (threadIdx.x == 0) P.ctl[1] = carry_sel;
}

// pick order: rank = selected entries with a larger gain, or the same gain in an earlier slot
__global__ void __launch_bounds__(128) k_pack_rank(pack_view P) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x, n = P.ctl[1];
    if (i >= n) return;
    const uint32_t p = P.sel[i];
    const unsigned long long g = P.egain[p];
    uint32_t r = 0;
    for (uint32_t j = 0; j < n; j++) {
        const uint32_t q = P.sel[j];
        const unsigned long long h = P.egain[q];
        r += (h > g || (h == g && q < p)) ? 1u : 0u;
    }
    P.ord[r] = p;
}

// one CTA: out_src_off[o] = constituents of the outputs before o (max_out + 1 entries; past n_out they repeat the total); n_out
__global__ void __launch_bounds__(1024) k_pack_offsets(pack_view P, uint32_t* out_src_off, uint32_t* n_out) {
    __shared__ uint32_t s_warp[32];
    const uint32_t n = P.ctl[1];
    uint32_t carry = 0;
    for (uint32_t b = 0; b < P.max_out; b += blockDim.x) {
        const uint32_t o = b + threadIdx.x;
        const uint32_t x = o < n ? P.fcnt[P.eslot[P.ord[o]]] : 0u;
        uint32_t total;
        const uint32_t ex = pack_block_scan(x, s_warp, &total);
        if (o < P.max_out) out_src_off[o] = carry + ex;
        carry += total;
    }
    if (threadIdx.x == 0) {
        out_src_off[P.max_out] = carry;
        *n_out = n;
    }
}

// CTA per output slot; slots past n_out are zero
__global__ void __launch_bounds__(128) k_pack_emit(pack_view P, const uint32_t* __restrict__ out_src_off, uint32_t* out_committee, uint32_t* out_data,
                                                   uint8_t* out_bits, unsigned long long* out_numerator, uint32_t* out_src) {
    const uint32_t o = blockIdx.x, n = P.ctl[1];
    uint8_t* ob = out_bits + (size_t)o * P.stride;
    if (o >= n) {
        for (uint32_t b = threadIdx.x; b < P.stride; b += blockDim.x) ob[b] = 0;
        if (threadIdx.x == 0) {
            out_committee[o] = 0;
            out_data[o] = 0;
            out_numerator[o] = 0;
        }
        return;
    }
    const uint32_t p = P.ord[o], q = P.eslot[p], k = P.cand_comm[P.list[q]];
    const uint32_t* row = P.frow + (size_t)q * P.wstride;
    for (uint32_t b = threadIdx.x; b < P.stride; b += blockDim.x) ob[b] = (uint8_t)(row[b >> 2] >> (8 * (b & 3)));
    if (threadIdx.x == 0) {
        out_committee[o] = k;
        out_data[o] = P.fdata[q];
        out_numerator[o] = P.egain[p];
    }
    if (threadIdx.x < 32) {                              // constituents in pool order: the committee's slots are sorted
        const uint32_t lane = threadIdx.x, end = P.off[k + 1];
        uint32_t base = out_src_off[o];
        for (uint32_t s0 = P.off[k]; s0 < end; s0 += 32) {
            const uint32_t s = s0 + lane;
            const bool hit = s < end && P.fold_of[s] == q;
            const uint32_t bal = __ballot_sync(B2_FULL_MASK, hit);
            if (hit) out_src[base + __popc(bal & ((1u << lane) - 1u))] = P.list[s];
            base += __popc(bal);
        }
    }
}

// the decompressed signatures of the constituents, contiguous in output order (the segments of k_g2_segment_sum)
__global__ void __launch_bounds__(128) k_pack_gather(const uint32_t* __restrict__ aff, const uint8_t* __restrict__ st, const uint32_t* __restrict__ src,
                                                     const uint32_t* __restrict__ total_p, uint32_t* gaff, uint8_t* gst) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= *total_p) return;
    const uint32_t c = src[i];
    const uint4* in = reinterpret_cast<const uint4*>(aff + 48 * (uint64_t)c);
    uint4* out = reinterpret_cast<uint4*>(gaff + 48 * (uint64_t)i);
#pragma unroll
    for (int k = 0; k < 12; k++) out[k] = in[k];
    gst[i] = st[c];
}

// an output with one constituent carries that signature's own bytes
__global__ void __launch_bounds__(128) k_pack_single(const uint8_t* __restrict__ sig96, const uint32_t* __restrict__ out_src_off,
                                                     const uint32_t* __restrict__ out_src, uint32_t max_out, uint8_t* out_sig96) {
    const uint32_t o = blockIdx.x * blockDim.x + threadIdx.x;
    if (o >= max_out || out_src_off[o + 1] - out_src_off[o] != 1) return;
    const uint8_t* s = sig96 + 96 * (uint64_t)out_src[out_src_off[o]];
#pragma unroll 1
    for (int b = 0; b < 96; b++) out_sig96[96 * (uint64_t)o + b] = s[b];
}

}  // namespace b2
