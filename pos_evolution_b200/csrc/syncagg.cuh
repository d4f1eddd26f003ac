// syncagg.cuh -- kernels of the sync-committee aggregate check (b2_sync_committee_load / b2_sync_aggregate_verify[_dev]): Altair
// process_sync_aggregate's eth_fast_aggregate_verify against committees that stay on the device for a whole period
// (pos-evolution.md:371-372, :540-590).
//
// The same committee_size keys sign every block of a period, so b2_sync_committee_load decodes and KeyValidates them once
// (k_g1_decompress_validate: affine records, the zero record and valid = 0 for a key that fails) and sums each committee's valid keys
// once (k_g1_segment_sum, one segment per committee).  The aggregate key of a block with k participants is then
//   k <= size / 2:  the sum of its participants' records,
//   k >  size / 2:  the committee sum plus the NEGATED records of its valid non-participants,
// whichever needs fewer additions: at 95 % participation of 512 keys about 26 mixed additions instead of about 490.
//
// k_sync_aggregate_pk: one WARP per block.  The bit row and the per-position valid bytes are read 32 positions at a time; a ballot
// compacts the positions that must be added (participants, or valid non-participants) into a per-warp list in shared memory, so the
// lanes then share ceil(m / 32) additions however the bits fall instead of one addition round per 32 positions.  The committee's
// records (48 KB at 512 keys) are read through L1 rather than staged: a block reads only the m records it adds, and every block of
// the batch reads the same table, which stays in L2.
// Status bits follow py_ecc FastAggregateVerify over the participants' keys: an invalid key matters only at a participating position,
// k == 0 is PK_EMPTY, a sum at infinity is PK_INFINITY; a committee index >= n_committees fails its block (PK_BAD_INDEX) and records
// GUARD_BAD_INDEX.  Output: the Jacobian key and status in the buffers K2 fills, so the pairing half of FastAggregateVerify follows as is.
//
// k_sync_empty_verdict: eth_fast_aggregate_verify's one difference from FastAggregateVerify -- with no participant the verdict is
// whether the signature is the G2 infinity encoding.
#pragma once
#include "kernels.cuh"

namespace b2 {

#define B2_SYNC_MAX_SIZE 1024         // committee_size limit: positions of one block's add list (u16) in shared memory
#define B2_SYNC_WARPS 4               // blocks (warps) per CTA

__global__ void __launch_bounds__(32 * B2_SYNC_WARPS) k_sync_aggregate_pk(const uint32_t* __restrict__ records, const uint8_t* __restrict__ valid,
                                                                           const uint32_t* __restrict__ sum_jac, uint32_t size, uint32_t n_comm,
                                                                           const uint32_t* __restrict__ cidx, const uint8_t* __restrict__ bits,
                                                                           uint32_t n, uint32_t* out_jac, uint8_t* out_status, uint32_t* guard) {
    __shared__ uint16_t list[B2_SYNC_WARPS][B2_SYNC_MAX_SIZE];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint32_t i = blockIdx.x * B2_SYNC_WARPS + warp;
    if (i >= n) return;
    const uint32_t c = cidx[i];
    if (c >= n_comm) {
        if (lane == 0) {
            if (guard) atomicOr(guard, (uint32_t)GUARD_BAD_INDEX);
            core_g1_finish(pt_inf<fp>(), PK_BAD_INDEX, 0, i, out_jac, out_status);
        }
        return;
    }
    const uint8_t* row = bits + (uint64_t)i * ((size + 7) >> 3);
    const uint8_t* vrow = valid + (uint64_t)c * size;
    uint32_t k = 0;
#pragma unroll 1
    for (uint32_t j = lane; j < size; j += 32) k += (row[j >> 3] >> (j & 7)) & 1u;
    k = __reduce_add_sync(B2_FULL_MASK, k);
    const bool complement = 2 * k > size;
    uint32_t m = 0, invalid = 0;
#pragma unroll 1
    for (uint32_t j0 = 0; j0 < size; j0 += 32) {
        const uint32_t j = j0 + lane;
        bool add = false;
        if (j < size) {
            const bool part = (row[j >> 3] >> (j & 7)) & 1u, ok = vrow[j] != 0;
            if (part && !ok) invalid = 1;
            add = ok && part != complement;
        }
        const unsigned mask = __ballot_sync(B2_FULL_MASK, add);
        if (add) list[warp][m + __popc(mask & ((1u << lane) - 1u))] = (uint16_t)j;
        m += __popc(mask);
    }
    __syncwarp();
    g1_jac acc = pt_inf<fp>();
    if (complement && lane == 0) acc = load_g1_jac(sum_jac + 36 * (uint64_t)c);
    const uint32_t* crec = records + 24 * (uint64_t)c * size;
#pragma unroll 1
    for (uint32_t t = lane; t < m; t += 32) {
        g1_aff p = load_record(crec, list[warp][t]);
        if (complement) p.y = fp_neg(p.y);
        acc = pt_add_mixed(acc, p);
    }
    // shuffle tree over the lanes that hold a partial sum (lane 0 and lanes < m): rounds whose partners are all empty are skipped
    const uint32_t live = max(min(m, 32u), 1u);
#pragma unroll 1
    for (uint32_t delta = 16; delta >= 1; delta >>= 1) {
        if (delta >= live) continue;
        g1_jac other = shfl_down_pod(acc, (int)delta);
        if ((uint32_t)lane < delta) acc = pt_add(acc, other);
    }
    invalid = __reduce_or_sync(B2_FULL_MASK, invalid);
    if (lane == 0) core_g1_finish(acc, invalid ? PK_INVALID_KEY : PK_OK, k, i, out_jac, out_status);
}

__global__ void __launch_bounds__(128) k_sync_empty_verdict(const uint8_t* __restrict__ pk_status, const uint8_t* __restrict__ sig96, uint32_t n,
                                                            uint8_t* ok) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n || pk_status[i] != (PK_EMPTY | PK_INFINITY)) return;      // k == 0 with a valid committee index
    const uint8_t* s = sig96 + 96 * (uint64_t)i;
    uint32_t rest = s[0] ^ 0xc0u;
#pragma unroll 1
    for (int b = 1; b < 96; b++) rest |= s[b];
    ok[i] = rest == 0;
}

}  // namespace b2
