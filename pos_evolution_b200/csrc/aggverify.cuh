// aggverify.cuh -- kernels of bls.AggregateVerify (b2_aggregate_verify / _pks / _dev): one signature over several (key, message)
// pairs, sets of any size back to back in one batch.  Per-item bodies and the item space: cores.cuh ("bls.AggregateVerify").
//   k_av_check   thread / set: the offsets start at 0, never decrease and stay inside the pairs (the _dev entry point cannot check
//                them on the host); otherwise every set of the call fails and GUARD_BAD_ROW is recorded
//   k_av_miller  thread / item: its Miller loop, then the block multiplies the values of each (block, set) run in shared memory and
//                the run's last item writes ONE value and status word to partial slot s + blockIdx.x
//   k_av_final   thread / set: the product of its partial slots, ONE final exponentiation, the verdict
// Partial slots are unique per run: runs (b, s) and (b', s') with b < b' and b + s = b' + s' would need s' < s while set s' still
// has an item in the later block b' -- impossible, sets are contiguous and in order.  So n_sets + n_blocks slots suffice.
#pragma once
#include "kernels.cuh"

namespace b2 {

// 64 items per block: their Miller values take 64 x 576 B = 36 KB of static shared memory, under the 48 KB a block gets without the
// dynamic shared-memory attribute (128 items would take 72 KB).  The kernel takes 255 registers (as k_miller), so registers, not shared
// memory, cap an SM at 8 warps for either size (4 blocks of 64 use 146 KB of shared memory): the smaller block costs no occupancy and
// halves the idle lanes of a batch's last block.
#define B2_AV_BLOCK 64

__global__ void __launch_bounds__(128) k_av_check(const uint32_t* __restrict__ pair_off, uint32_t n_sets, uint64_t n_pairs, uint32_t* bad_row,
                                                  uint32_t* guard) {
    const uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n_sets) return;
    const uint32_t o0 = pair_off[s], o1 = pair_off[s + 1];
    if (o1 < o0 || (s == 0 && o0 != 0) || (s == n_sets - 1 && o1 > n_pairs)) {
        atomicOr(bad_row, 1u);
        if (guard) atomicOr(guard, (uint32_t)GUARD_BAD_ROW);
    }
}

// signer == nullptr: pair j uses key record j (explicit keys, decoded by k_g1_decompress_validate); else record signer[j] of a table of
// n_keys (the registry).  The grid covers n_pairs + n_sets items; those past pair_off[n_sets] + n_sets are idle.
__global__ void __launch_bounds__(B2_AV_BLOCK) k_av_miller(const uint32_t* __restrict__ pair_off, uint32_t n_sets, const uint32_t* __restrict__ signer,
                                                           const uint32_t* __restrict__ records, const uint8_t* __restrict__ valid, uint64_t n_keys,
                                                           const uint32_t* __restrict__ h_aff, const uint8_t* __restrict__ hflag,
                                                           const uint32_t* __restrict__ s_aff, const uint8_t* __restrict__ sflag,
                                                           const uint32_t* __restrict__ bad_row, uint32_t* f_part, uint32_t* st_part, uint32_t* guard) {
    __shared__ fp12 sf[B2_AV_BLOCK];
    __shared__ uint32_t sst[B2_AV_BLOCK], sset[B2_AV_BLOCK];
    if (*bad_row) return;                     // malformed offsets: k_av_final fails every set; nothing the offsets point at is read
    constexpr uint32_t IDLE = 0xffffffffu;
    const uint32_t t = threadIdx.x, i = blockIdx.x * B2_AV_BLOCK + t;
    uint32_t bad = 0, s = IDLE;
    g1_jac p = pt_inf<fp>();
    g2_aff q;
    q.x = fp2_zero();
    q.y = fp2_zero();
    bool q_inf = true;
    if (i < pair_off[n_sets] + n_sets) {
        s = av_set_of(pair_off, n_sets, i);
        const uint32_t j = i - s;                 // pair j of the set, or pair_off[s+1] for its signature item
        if (j < pair_off[s + 1]) {
            core_av_pair(records, valid, signer ? signer[j] : j, n_keys, load_g2_aff(h_aff + 48 * (uint64_t)j), hflag[j], p, q, q_inf, bad);
        } else {
            core_av_sig(load_g2_aff(s_aff + 48 * (uint64_t)s), sflag[s], p, q, q_inf, bad);
        }
    }
    if ((bad & AV_BAD_INDEX) && guard) atomicOr(guard, (uint32_t)GUARD_BAD_INDEX);
    fp12 f = miller_loop(p, q, q_inf);
    sf[t] = f;
    sst[t] = bad;
    sset[t] = s;
    __syncthreads();
    // segmented inclusive scan of the products (Fp12 multiplication commutes, so the order does not matter): after the round with
    // distance d, item t holds the product of the last min(2d, run length so far) items of its run up to t
#pragma unroll 1
    for (uint32_t d = 1; d < B2_AV_BLOCK; d <<= 1) {
        const bool take = s != IDLE && t >= d && sset[t - d] == s;
        fp12 o;
        uint32_t ob = 0;
        if (take) {
            o = sf[t - d];
            ob = sst[t - d];
        }
        __syncthreads();
        if (take) {
            f = fp12_mul(f, o);
            bad |= ob;
            sf[t] = f;
            sst[t] = bad;
        }
        __syncthreads();
    }
    if (s != IDLE && (t == B2_AV_BLOCK - 1 || sset[t + 1] != s)) {      // the last item of its (block, set) run
        const uint64_t slot = (uint64_t)s + blockIdx.x;
        uint32_t* o = f_part + 144 * slot;
        const uint32_t* w = reinterpret_cast<const uint32_t*>(&f);
#pragma unroll 1
        for (int k = 0; k < 144; k++) o[k] = w[k];
        st_part[slot] = bad;
    }
}

__global__ void __launch_bounds__(32) k_av_final(const uint32_t* __restrict__ pair_off, uint32_t n_sets, const uint32_t* __restrict__ bad_row,
                                                 const uint32_t* __restrict__ f_part, const uint32_t* __restrict__ st_part, uint8_t* ok) {
    const uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n_sets) return;
    if (*bad_row) {
        ok[s] = 0;
        return;
    }
    const uint32_t b0 = (pair_off[s] + s) / B2_AV_BLOCK, b1 = (pair_off[s + 1] + s) / B2_AV_BLOCK;     // blocks of its first and last item
    fp12 F;
    uint32_t* w = reinterpret_cast<uint32_t*>(&F);
    const uint32_t* p = f_part + 144 * ((uint64_t)s + b0);
#pragma unroll 1
    for (int k = 0; k < 144; k++) w[k] = p[k];
    uint32_t bad = st_part[s + b0];
#pragma unroll 1
    for (uint32_t b = b0 + 1; b <= b1; b++) {
        fp12 m;
        uint32_t* wm = reinterpret_cast<uint32_t*>(&m);
        const uint32_t* pm = f_part + 144 * ((uint64_t)s + b);
#pragma unroll 1
        for (int k = 0; k < 144; k++) wm[k] = pm[k];
        F = fp12_mul(F, m);
        bad |= st_part[s + b];
    }
    ok[s] = core_av_verdict(F, bad, pair_off[s + 1] > pair_off[s]);
}

}  // namespace b2
