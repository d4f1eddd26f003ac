// slasher.cuh -- detection of slashable attestations (is_slashable_attestation_data, pos-evolution.md:1128-1143): the double and
// surround votes of every accepted aggregate, from per-validator span tables over a ring of H epochs.  Included by b200pos.cu only.
//
// Tables, validator-major (cell (v, e) at (v - v_begin) * H + e mod H; the walks below run along e for one validator).  A slasher may
// hold a range [v_begin, v_begin + n_rows) of the n_val validators only (one rank's share of a sharded registry): members outside it
// are skipped without a guard bit, while everything per aggregate (status, id, column count, root log) is the same on every range.
//   min_span u16: min over the accepted attestations (s, t) of v with s > e of t - e; none = SL_NONE
//   max_span u16: max over those with s < e < t of t - e;                      none = 0
//   first_id u16: id of the first accepted attestation of v with target e;     none = SL_NONE
// and per target column a log of the data roots of its accepted aggregates, root[e mod H][id], ids in acceptance order.
// With them "attestation (s, t) of v surrounds an earlier one" is s + min_span[v][s] < t, "is surrounded by one" is
// s + max_span[v][s] > t, and "double vote" is root[t][first_id[v][t]] != its own root: a constant number of cells per member.
//
// Exact against everything ever accepted, although columns are recycled: an attestation is accepted only when low <= s <= t <= cur,
// column e exists from the moment e is current, every attestation with source > e or target >= e is accepted after that moment,
// and the window only moves up.  So when an attestation conflicting with a later accepted (s, t) was recorded, columns s and t
// already existed, lay inside its walk, and have not been recycled since.
#pragma once
#include <stdint.h>

#include "kernels.cuh"

namespace b2 {

constexpr uint32_t SL_NONE = 0xffffu;            // empty min_span / first_id cell; aggregate without an id
enum SlasherStatus : int32_t {
    SL_OK = 0,
    SL_NOT_ACCEPTED = 1,       // accept[a] == 0
    SL_SOURCE_AFTER_TARGET = 2,
    SL_TARGET_AHEAD = 3,       // target > current epoch
    SL_SOURCE_EXPIRED = 4,     // source below the window
    SL_COLUMN_FULL = 5,        // max_attestations_per_target aggregates with this target are recorded already
    SL_BAD_ROW = 6             // device form only: offsets run backwards or the row exceeds the bit row (GUARD_BAD_ROW)
};
enum SlasherKind : uint8_t { SL_DOUBLE = 1, SL_SURROUNDS = 2, SL_SURROUNDED = 4 };

struct slasher_view {
    uint16_t *min_span, *max_span, *first_id;      // u16[n_val][H]
    uint32_t* count;                               // u32[H] aggregates recorded per target column
    uint8_t* root;                                 // u8[H][K][32]
    uint64_t n_val, n_rows;                        // validators of the registry; rows held: v_begin .. v_begin + n_rows - 1
    uint32_t v_begin, H, K, cur, low;
};

// 16-bit atomic min / max: a CAS loop that issues nothing when the cell already holds a value at least as good; returns the value
// seen before
__device__ __forceinline__ uint32_t sl_atomic_min(uint16_t* p, uint32_t val) {
    unsigned short old = *(volatile unsigned short*)p;
    while (val < old) {
        const unsigned short seen = atomicCAS((unsigned short*)p, old, (unsigned short)val);
        if (seen == old) break;
        old = seen;
    }
    return old;
}
__device__ __forceinline__ uint32_t sl_atomic_max(uint16_t* p, uint32_t val) {
    unsigned short old = *(volatile unsigned short*)p;
    while (val > old) {
        const unsigned short seen = atomicCAS((unsigned short*)p, old, (unsigned short)val);
        if (seen == old) break;
        old = seen;
    }
    return old;
}

// status of aggregate a before ids are assigned (everything but SL_COLUMN_FULL); a function of the call's inputs and the window alone
__device__ __forceinline__ int32_t sl_row_status(const slasher_view& S, const uint32_t* off, uint32_t stride, const uint64_t* source_epoch,
                                                 const uint64_t* target_epoch, const uint8_t* accept, uint32_t a) {
    if (accept && !accept[a]) return SL_NOT_ACCEPTED;
    const uint32_t o0 = off[a], o1 = off[a + 1];
    if (o1 < o0 || o1 - o0 > stride * 8u) return SL_BAD_ROW;
    const uint64_t s = source_epoch[a], t = target_epoch[a];
    if (s > t) return SL_SOURCE_AFTER_TARGET;
    if (t > S.cur) return SL_TARGET_AHEAD;
    if (s < S.low) return SL_SOURCE_EXPIRED;
    return SL_OK;
}

// Thread per aggregate: status, id and the root into the column's log.  id = aggregates the column held before the call + the rank of
// a among the acceptable aggregates of the call with the same target, by position: a function of the call, not of scheduling.  The
// rank is counted against every earlier aggregate, 128 at a time: the block derives their statuses once into shared memory and each
// thread compares its target with the tile (quadratic in n_agg, a few thousand per call, but a broadcast read per comparison).  The
// column counts are only read here; k_slasher_record raises them.
__global__ void __launch_bounds__(128) k_slasher_rows(slasher_view S, const uint32_t* __restrict__ off, uint32_t stride,
                                                       const uint64_t* __restrict__ source_epoch, const uint64_t* __restrict__ target_epoch,
                                                       const uint8_t* __restrict__ root32, const uint8_t* __restrict__ accept, uint32_t n_agg,
                                                       int32_t* status_out, uint32_t* agg_id, uint32_t* guard) {
    __shared__ uint32_t tile[128];      // target of an acceptable aggregate (< 2^32 - 1, as cur is), else 0xffffffff
    const uint32_t a = blockIdx.x * 128 + threadIdx.x;
    int32_t st = a < n_agg ? sl_row_status(S, off, stride, source_epoch, target_epoch, accept, a) : (int32_t)SL_NOT_ACCEPTED;
    const uint32_t t = st == SL_OK ? (uint32_t)target_epoch[a] : 0;
    uint32_t rank = 0;
    for (uint32_t base = 0; base <= blockIdx.x * 128; base += 128) {
        const uint32_t b = base + threadIdx.x;
        tile[threadIdx.x] = b < n_agg && sl_row_status(S, off, stride, source_epoch, target_epoch, accept, b) == SL_OK ? (uint32_t)target_epoch[b] : 0xffffffffu;
        __syncthreads();
        const uint32_t n_before = st == SL_OK ? min(128u, a - base) : 0;
        for (uint32_t k = 0; k < n_before; k++) rank += tile[k] == t;
        __syncthreads();
    }
    if (a >= n_agg) return;
    uint32_t id = SL_NONE;
    if (st == SL_BAD_ROW && guard) atomicOr(guard, (uint32_t)GUARD_BAD_ROW);
    if (st != SL_NOT_ACCEPTED && st != SL_BAD_ROW && (source_epoch[a] >= 0xffffffffull || target_epoch[a] >= 0xffffffffull) && guard)
        atomicOr(guard, (uint32_t)GUARD_BAD_EPOCH);      // such a row is SL_SOURCE_AFTER_TARGET or SL_TARGET_AHEAD: cur fits 32 bits
    if (st == SL_OK) {
        const uint32_t col = t % S.H;
        const uint64_t want = (uint64_t)S.count[col] + rank;
        if (want >= S.K) {
            st = SL_COLUMN_FULL;
        } else {
            id = (uint32_t)want;
            uint8_t* dst = S.root + 32 * ((uint64_t)col * S.K + id);      // bytewise: the caller's roots need no alignment
            for (int k = 0; k < 32; k++) dst[k] = root32[32 * (uint64_t)a + k];
        }
    }
    status_out[a] = st;
    agg_id[a] = id;
}

// selected member j of aggregate a -> its row v - v_begin of the tables; false for a clear bit, an index outside the registry
// (GUARD_BAD_INDEX) or a validator outside this slasher's range (silently: another range holds it)
__device__ __forceinline__ bool sl_member(const slasher_view& S, const uint32_t* members, uint32_t o0, const uint8_t* bits, uint32_t stride,
                                          uint32_t a, uint32_t j, uint32_t& row, uint32_t* guard) {
    if (!((bits[(uint64_t)a * stride + (j >> 3)] >> (j & 7)) & 1)) return false;
    const uint32_t v = members[o0 + j];
    if (v >= S.n_val) {
        if (guard) atomicOr(guard, (uint32_t)GUARD_BAD_INDEX);
        return false;
    }
    row = v - S.v_begin;      // wraps above n_rows for v < v_begin
    return row < S.n_rows;
}

// Block per accepted aggregate (s, t), thread per member: first_id by atomic min on the id, then the two span walks.
__global__ void __launch_bounds__(128) k_slasher_record(slasher_view S, const uint32_t* __restrict__ members, const uint32_t* __restrict__ off,
                                                         const uint8_t* __restrict__ bits, uint32_t stride,
                                                         const uint64_t* __restrict__ source_epoch, const uint64_t* __restrict__ target_epoch,
                                                         const uint32_t* __restrict__ agg_id, uint32_t n_agg, uint32_t* guard) {
    const uint32_t a = blockIdx.x;
    if (a >= n_agg) return;
    const uint32_t id = agg_id[a];
    if (id == SL_NONE) return;
    const uint32_t s = (uint32_t)source_epoch[a], t = (uint32_t)target_epoch[a], H = S.H;
    const uint32_t cs = s % H, ct = t % H, o0 = off[a], size = off[a + 1] - o0;
    if (threadIdx.x == 0) atomicMax(&S.count[ct], id + 1);
    for (uint32_t j = threadIdx.x; j < size; j += blockDim.x) {
        uint32_t v;
        if (!sl_member(S, members, o0, bits, stride, a, j, v, guard)) continue;
        const uint64_t base = (uint64_t)v * H;
        sl_atomic_min(S.first_id + base + ct, id);
        // min_span: columns e = s-1 down to low see target t at distance t - e.  The smallest target seen from a column can only
        // fall towards lower e (more sources lie above it), so a cell that already holds a value <= ours was written for a target
        // <= t, and whoever wrote it covers, or has covered, every lower column with a value at least as small: stop there.  That
        // holds under concurrency too, because the other writer finishes its own walk (or stops at a still smaller one, and so on).
        uint32_t p = cs, d = t - s;
        for (uint32_t e = s; e > S.low; e--) {
            p = p ? p - 1 : H - 1;
            d++;
            if (sl_atomic_min(S.min_span + base + p, d) <= d) break;
        }
        // max_span: columns e = s+1 up to t-1 lie strictly inside (s, t) at distance t - e.  A cell that already holds a value >= ours
        // was written for a target >= t by a walk that continues up to that target: stop there, by the mirrored argument.
        p = cs;
        d = t - s;
        for (uint32_t e = s + 1; e < t; e++) {
            p = p + 1 == H ? 0 : p + 1;
            d--;
            if (sl_atomic_max(S.max_span + base + p, d) >= d) break;
        }
    }
}

// Same mapping, after k_slasher_record of the same call has finished: kind byte and the two conflicting targets of every member slot
// of every well-formed row (0 / none for clear bits and rows that were not accepted); flagged slots are counted with one atomic per
// warp.  An attestation's own record cannot trip its own check: its source is neither > s nor < s and its root equals itself.
__global__ void __launch_bounds__(128) k_slasher_check(slasher_view S, const uint32_t* __restrict__ members, const uint32_t* __restrict__ off,
                                                        const uint8_t* __restrict__ bits, uint32_t stride,
                                                        const uint64_t* __restrict__ source_epoch, const uint64_t* __restrict__ target_epoch,
                                                        const uint32_t* __restrict__ agg_id, uint32_t n_agg, uint8_t* kind_out,
                                                        uint32_t* conflict_out, uint32_t* n_flagged) {
    const uint32_t a = blockIdx.x;
    if (a >= n_agg) return;
    const uint32_t id = agg_id[a], H = S.H, o0 = off[a], size = off[a + 1] - o0;
    if (off[a + 1] < o0 || size > stride * 8u) return;      // a malformed row has no member slots to write (its status says why)
    const uint32_t s = (uint32_t)source_epoch[a], t = (uint32_t)target_epoch[a];
    const uint32_t cs = id == SL_NONE ? 0 : s % H, ct = id == SL_NONE ? 0 : t % H;
    const uint8_t* log = S.root + 32 * (uint64_t)ct * S.K;
    for (uint32_t j0 = 0; j0 < size; j0 += blockDim.x) {      // whole warps iterate, for the ballot
        const uint32_t j = j0 + threadIdx.x;
        uint32_t kind = 0, c_min = 0xffffffffu, c_max = 0xffffffffu, v;
        if (j < size && id != SL_NONE && sl_member(S, members, o0, bits, stride, a, j, v, nullptr)) {
            const uint64_t base = (uint64_t)v * H;
            const uint32_t first = S.first_id[base + ct];
            if (first != id) {
                const uint4* x = reinterpret_cast<const uint4*>(log + 32 * (uint64_t)first);
                const uint4* y = reinterpret_cast<const uint4*>(log + 32 * (uint64_t)id);
                const uint4 x0 = x[0], x1 = x[1], y0 = y[0], y1 = y[1];
                if ((x0.x ^ y0.x) | (x0.y ^ y0.y) | (x0.z ^ y0.z) | (x0.w ^ y0.w) | (x1.x ^ y1.x) | (x1.y ^ y1.y) | (x1.z ^ y1.z) | (x1.w ^ y1.w))
                    kind |= SL_DOUBLE;
            }
            const uint32_t lo = S.min_span[base + cs], hi = S.max_span[base + cs];
            if (lo != SL_NONE && s + lo < t) kind |= SL_SURROUNDS, c_min = s + lo;
            if (s + hi > t) kind |= SL_SURROUNDED, c_max = s + hi;
        }
        if (j < size) {
            kind_out[o0 + j] = (uint8_t)kind;
            if (conflict_out) {
                conflict_out[2 * (uint64_t)(o0 + j)] = c_min;
                conflict_out[2 * (uint64_t)(o0 + j) + 1] = c_max;
            }
        }
        const unsigned flagged = __ballot_sync(B2_FULL_MASK, kind != 0);
        if (flagged && (threadIdx.x & 31) == 0) atomicAdd(n_flagged, (uint32_t)__popc(flagged));
    }
}

// Equivocation discounting (pos-evolution.md:1405-1461): thread per member slot of an update (after its k_slasher_check).  A flagged
// slot (kind != 0) marks its validator in the registry's equivocating table, so that from then on it neither moves its latest message
// (k_lmd_phase1/2) nor counts in a head.  Marks are set by atomicOr on the aligned 32-bit word holding v's byte (the table is padded to
// whole words), so exactly one slot -- the one that turned v's byte from 0 to nonzero -- reports v as newly marked, however many slots
// flag v and whether or not v was marked before; newly marked slots are counted with one atomic per warp.  Only validators of the
// slasher's rows [v_begin, v_begin + n_rows) can be flagged; the range test keeps a stray kind byte outside it from marking anything.
__global__ void __launch_bounds__(256) k_slasher_discount(const uint32_t* __restrict__ members, const uint8_t* __restrict__ kind, uint64_t n_slots,
                                                           uint64_t n_val, uint32_t v_begin, uint64_t n_rows, uint8_t* equiv, uint8_t* new_out,
                                                           uint32_t* n_new) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    bool fresh = false;
    if (i < n_slots) {
        const uint32_t v = kind[i] ? members[i] : 0xffffffffu;
        if (v < n_val && (uint32_t)(v - v_begin) < n_rows) {
            const uint32_t shift = 8u * (v & 3u);
            const uint32_t old = atomicOr(reinterpret_cast<uint32_t*>(equiv + (v & ~3u)), 1u << shift);
            fresh = ((old >> shift) & 0xffu) == 0;
        }
        new_out[i] = fresh;
    }
    const unsigned m = __ballot_sync(B2_FULL_MASK, fresh);
    if (m && (threadIdx.x & 31) == 0) atomicAdd(n_new, (uint32_t)__popc(m));
}

// Thread per validator of a range [v_begin, v_begin + n): equiv[v] |= table[v - v_begin] -- one rank's slice of the equivocating table
// merged into another rank's replica (sharded epochs).  A byte has one writer, so no atomics.
__global__ void __launch_bounds__(256) k_equiv_merge(const uint8_t* __restrict__ table, uint64_t v_begin, uint64_t n, uint8_t* equiv) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n && table[i]) equiv[v_begin + i] |= table[i];
}

// The window moves up: the columns of the epochs first .. first + n_cols - 1 (n_cols < H) become empty
__global__ void __launch_bounds__(256) k_slasher_advance(slasher_view S, uint32_t first, uint32_t n_cols) {
    const uint64_t total = S.n_rows * n_cols;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (uint64_t)gridDim.x * blockDim.x) {
        const uint64_t cell = (i / n_cols) * S.H + (first + (uint32_t)(i % n_cols)) % S.H;
        S.min_span[cell] = (uint16_t)SL_NONE;
        S.max_span[cell] = 0;
        S.first_id[cell] = (uint16_t)SL_NONE;
    }
    if (blockIdx.x == 0)
        for (uint32_t c = threadIdx.x; c < n_cols; c += blockDim.x) S.count[(first + c) % S.H] = 0;
}

}  // namespace b2
