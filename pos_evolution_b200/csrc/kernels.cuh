// kernels.cuh -- the __global__ kernels of libb200pos.so (sm_90a).  Per-thread bodies live in
// cores.cuh (shared with the host-sim tests); this file adds thread mapping, warp-shuffle /
// shared-memory tree reductions of partial EC points, and the fork-choice kernels K7-K9.
// Kernel numbering follows SURVEY.md section 2.
#pragma once
#include <cuda_runtime.h>

#include "cores.cuh"

#ifndef B2_TAIL_MIN_BLOCKS
#define B2_TAIL_MIN_BLOCKS 1 /* 4 (a 128-register cap, the footprint of one decompression block) measured slower: 40.8 vs 39.8 ms */
#endif
namespace b2 {

#define B2_FULL_MASK 0xffffffffu

template <class T> __device__ __forceinline__ T shfl_down_pod(const T& v, int delta) {
    constexpr int W = sizeof(T) / 4;
    T r;
    const uint32_t* s = reinterpret_cast<const uint32_t*>(&v);
    uint32_t* d = reinterpret_cast<uint32_t*>(&r);
#pragma unroll
    for (int i = 0; i < W; i++) d[i] = __shfl_down_sync(B2_FULL_MASK, s[i], delta);
    return r;
}

// Sum of the per-thread partial points of a block; result valid in thread 0.  Warp level: shuffle
// tree (5 rounds of Jacobian additions); across warps: shared memory.  `smem` holds blockDim/32 points.
template <class F> __device__ __forceinline__ jac<F> block_sum_points(jac<F> acc, jac<F>* smem) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarp = blockDim.x >> 5;
#pragma unroll 1
    for (int delta = 16; delta >= 1; delta >>= 1) {
        jac<F> other = shfl_down_pod(acc, delta);
        if (lane < delta) acc = pt_add(acc, other);
    }
    if (lane == 0) smem[warp] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
#pragma unroll 1
        for (int w = 1; w < nwarp; w++) acc = pt_add(acc, smem[w]);
    }
    return acc;
}

// ------------------------------------------------------------------------------------------ registry
__global__ void __launch_bounds__(128) k_registry_load(const uint8_t* __restrict__ pk48, uint64_t n, uint32_t* records, uint8_t* valid) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) core_registry_load(pk48, records, valid, i);
}

// ------------------------------------------------------------------------------------------ device-side input guards
// The *_dev entry points take device pointers, which the host cannot validate (b2_fast_aggregate_verify & co. do: check_batch).
// Every kernel that follows caller-supplied indices therefore checks them itself: a committee row whose offsets run backwards or
// whose size exceeds the bit row, a member index >= n_val, or a target epoch that does not fit the 32-bit key field is SKIPPED
// (the aggregate then fails verification / contributes nothing) and recorded in the context's guard word (b2_guard_flags).
enum GuardBits : uint32_t { GUARD_BAD_INDEX = 1, GUARD_BAD_ROW = 2, GUARD_BAD_EPOCH = 4, GUARD_BAD_POOL = 8 /* pack.cuh */ };
__device__ __forceinline__ uint32_t guarded_row_size(const uint32_t* off, uint32_t a, uint32_t bits_stride, uint32_t* guard) {
    const uint32_t o0 = off[a], o1 = off[a + 1];
    if (o1 < o0 || o1 - o0 > bits_stride * 8u) {
        if (threadIdx.x == 0 && guard) atomicOr(guard, (uint32_t)GUARD_BAD_ROW);
        return 0xffffffffu;
    }
    return o1 - o0;
}

// ------------------------------------------------------------------------------------------ K2: G1 gather + aggregate
// one block per aggregate; thread t takes members t, t+B, ...: bit test, index load, 96-byte record
// gather (six 128-bit loads), mixed addition; then the block-level tree.
__global__ void __launch_bounds__(128) k_g1_aggregate(const uint32_t* __restrict__ records, const uint8_t* __restrict__ valid,
                                                       const uint32_t* __restrict__ members, const uint32_t* __restrict__ off,
                                                       const uint8_t* __restrict__ bits, uint32_t bits_stride, uint32_t n_agg,
                                                       uint32_t* out_jac, uint8_t* out_status, uint64_t n_val, uint32_t* guard) {
    __shared__ g1_jac red[4];
    const uint32_t a = blockIdx.x;
    if (a >= n_agg) return;
    uint32_t size = guarded_row_size(off, a, bits_stride, guard);
    g1_jac acc = pt_inf<fp>();
    uint32_t status = 0, cnt = 0;
    const bool row_bad = size == 0xffffffffu;
    if (row_bad) {
        size = 0;
        status = PK_BAD_INDEX;
    }
#pragma unroll 1
    for (uint32_t j = threadIdx.x; j < size; j += blockDim.x)
        core_g1_accumulate(records, valid, members, off, bits, bits_stride, a, j, acc, status, cnt, n_val);
    acc = block_sum_points(acc, red);
    status = __syncthreads_or((int)status);
    cnt = __syncthreads_count(cnt != 0);
    if (threadIdx.x == 0) {
        if ((status & PK_BAD_INDEX) && !row_bad && guard) atomicOr(guard, (uint32_t)GUARD_BAD_INDEX);
        core_g1_finish(acc, status, cnt, a, out_jac, out_status);
    }
}

// Jacobian aggregated pubkeys -> compressed 48 bytes (only for the b2_g1_aggregate entry point)
__global__ void __launch_bounds__(64) k_g1_compress(const uint32_t* __restrict__ jac_in, uint32_t n, uint8_t* out48) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) g1_compress(load_g1_jac(jac_in + 36 * (uint64_t)i), out48 + 48 * (uint64_t)i);
}

// pyspec-literal form: decompress + KeyValidate explicit pubkeys, then sum per aggregate
__global__ void __launch_bounds__(128) k_g1_decompress_validate(const uint8_t* __restrict__ pk48, uint64_t n, uint32_t* records, uint8_t* valid) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) core_registry_load(pk48, records, valid, i);
}
__global__ void __launch_bounds__(128) k_g1_segment_sum(const uint32_t* __restrict__ records, const uint8_t* __restrict__ valid,
                                                         const uint32_t* __restrict__ off, uint32_t n_agg, uint32_t* out_jac, uint8_t* out_status) {
    __shared__ g1_jac red[4];
    const uint32_t a = blockIdx.x;
    if (a >= n_agg) return;
    g1_jac acc = pt_inf<fp>();
    uint32_t status = 0, cnt = 0;
#pragma unroll 1
    for (uint32_t j = off[a] + threadIdx.x; j < off[a + 1]; j += blockDim.x) {
        cnt++;
        if (!valid[j]) {
            status |= PK_INVALID_KEY;
        } else {
            acc = pt_add_mixed(acc, load_record(records, j));
        }
    }
    acc = block_sum_points(acc, red);
    status = __syncthreads_or((int)status);
    cnt = __syncthreads_count(cnt != 0);
    if (threadIdx.x == 0) core_g1_finish(acc, status, cnt, a, out_jac, out_status);
}

// ------------------------------------------------------------------------------------------ K3: bls.Aggregate
// stage 1: one thread per signature: ZCash decode + Fp2 square root (two Fp exponentiations) -> affine point
__global__ void __launch_bounds__(128, 4) k_g2_decompress(const uint8_t* __restrict__ sig96, uint64_t n, uint32_t* aff_out, uint8_t* st_out) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    g2_aff s;
    s.x = fp2_zero();
    s.y = fp2_zero();
    int st = g2_decompress(sig96 + 96 * i, s);
    uint4* o = reinterpret_cast<uint4*>(aff_out + 48 * i);
    const uint32_t* w = reinterpret_cast<const uint32_t*>(&s);
#pragma unroll
    for (int k = 0; k < 12; k++) o[k] = make_uint4(w[4 * k], w[4 * k + 1], w[4 * k + 2], w[4 * k + 3]);
    st_out[i] = (uint8_t)st;
}
// stage 2: one WARP per segment (each lane adds every 32nd point, then a 5-round shuffle tree) -> Jacobian sum (72 words) + status.  The inversion needed for
// the compressed encoding is NOT done here (127 threads would idle behind it): stage 3 does it with a thread per segment.
__global__ void __launch_bounds__(32) k_g2_segment_sum(const uint32_t* __restrict__ aff, const uint8_t* __restrict__ st,
                                                            const uint32_t* __restrict__ seg_off, uint32_t n_seg, uint32_t* sum_jac,
                                                            int32_t* seg_status, uint64_t n_sig, uint32_t* guard) {
    __shared__ g2_jac red[4];
    const uint32_t s = blockIdx.x;
    if (s >= n_seg) return;
    uint32_t begin = seg_off[s], end = seg_off[s + 1];
    g2_jac acc = pt_inf<fp2>();
    uint32_t bad = 0;
    if (end < begin || end > n_sig) {           // malformed offsets (device-pointer entry points): the segment is undecodable, nothing is read
        if (threadIdx.x == 0 && guard) atomicOr(guard, (uint32_t)GUARD_BAD_ROW);
        begin = end = 0;
        bad = 1;
    }
#pragma unroll 1
    for (uint32_t j = begin + threadIdx.x; j < end; j += blockDim.x) {
        uint8_t f = st[j];
        if (f == DEC_BAD) {
            bad = 1;
        } else if (f == DEC_OK) {
            g2_aff p;
            const uint4* in = reinterpret_cast<const uint4*>(aff + 48 * (uint64_t)j);
            uint32_t* w = reinterpret_cast<uint32_t*>(&p);
#pragma unroll
            for (int k = 0; k < 12; k++) {
                uint4 v = in[k];
                w[4 * k] = v.x; w[4 * k + 1] = v.y; w[4 * k + 2] = v.z; w[4 * k + 3] = v.w;
            }
            acc = pt_add_mixed(acc, p);
        }
    }
    acc = block_sum_points(acc, red);
    bad = __syncthreads_or((int)bad);
    if (threadIdx.x == 0) {
        seg_status[s] = bad ? 1 : (end == begin ? 2 : 0);
        uint32_t* o = sum_jac + 72 * (uint64_t)s;
        const uint32_t* w = reinterpret_cast<const uint32_t*>(&acc);
#pragma unroll 1
        for (int k = 0; k < 72; k++) o[k] = w[k];
    }
}
// stage 3: one thread per segment: Jacobian sum -> affine (one Fp2 inversion) -> compressed 96 bytes (bls.Aggregate's result).
// When `s_aff` is given (epoch pipeline) the affine point and its signature flag are handed to the verification stage
// directly -- compress followed by decompress is the identity, so the Fp2 square root of the aggregate is skipped -- and
// the G2 subgroup check FastAggregateVerify performs on the signature is done here.
__global__ void __launch_bounds__(128, B2_TAIL_MIN_BLOCKS) k_g2_finish(const uint32_t* __restrict__ sum_jac, const int32_t* __restrict__ seg_status, uint32_t n_seg,
                                                   uint8_t* out96, uint32_t* s_aff, uint8_t* sflag) {
    uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n_seg) return;
    g2_jac acc;
    uint32_t* w = reinterpret_cast<uint32_t*>(&acc);
    const uint32_t* in = sum_jac + 72 * (uint64_t)s;
#pragma unroll 1
    for (int k = 0; k < 72; k++) w[k] = in[k];
    const int32_t st = seg_status[s];
    g2_aff a;
    a.x = fp2_zero();
    a.y = fp2_zero();
    bool finite = (st == 0) && pt_to_affine(acc, a);
    uint8_t* o = out96 + 96 * (uint64_t)s;
    if (st != 0) {
#pragma unroll 1
        for (int k = 0; k < 96; k++) o[k] = 0;
    } else {
        g2_compress_affine(a, !finite, o);
    }
    if (s_aff) {
        uint8_t f = (st != 0) ? SIG_INVALID : (!finite ? SIG_INFINITY : (g2_in_subgroup(pt_from_affine(a)) ? SIG_OK : SIG_INVALID));
        uint32_t* oa = s_aff + 48 * (uint64_t)s;
        const uint32_t* wa = reinterpret_cast<const uint32_t*>(&a);
#pragma unroll 1
        for (int k = 0; k < 48; k++) oa[k] = wa[k];
        sflag[s] = f;
    }
}

// ------------------------------------------------------------------------------------------ K4-K6: verification pipeline
// Two lanes per message: hash_to_curve maps TWO field elements to the curve (RFC 9380 section 3: Q0 = map(u0), Q1 = map(u1)) with
// three Fp exponentiations each, independent of one another -- the odd lane maps u1 while the even lane maps u0 and then takes Q1 over
// by shuffle for the addition, the cofactor clearing and the affine conversion.  Same functions, same bytes as core_hash_msg; the
// critical path of the kernel (one thread's instruction stream: 6.3 ms for 2 048 messages) loses one of its two SSWU maps.
__global__ void __launch_bounds__(128, B2_TAIL_MIN_BLOCKS) k_hash_to_g2(const uint8_t* __restrict__ msg32, uint32_t n, uint32_t* h_aff, uint8_t* hflag) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t a = t >> 1, half = t & 1u;
    const bool live = a < n;
    g2_jac q = pt_inf<fp2>();
    if (live) {
        uint8_t dst[B2_DST_POP_LEN];
#pragma unroll 1
        for (int i = 0; i < B2_DST_POP_LEN; i++) dst[i] = dst_pop_byte(i);
        fp2 u0, u1;
        hash_to_field_fp2x2(msg32 + 32 * (uint64_t)a, 32, dst, B2_DST_POP_LEN, u0, u1);
        q = map_to_curve_g2(half ? u1 : u0);
    }
    const g2_jac other = shfl_down_pod(q, 1);               // the odd lane's Q1 (whole warps execute this: blockDim is a multiple of 32)
    if (!live || half) return;
    q = g2_clear_cofactor(pt_add(q, other));
    g2_aff h;
    h.x = fp2_zero();
    h.y = fp2_zero();
    const uint8_t f = pt_to_affine(q, h) ? 0 : 1;
    uint32_t* o = h_aff + 48 * (uint64_t)a;
    const uint32_t* w = reinterpret_cast<const uint32_t*>(&h);
#pragma unroll
    for (int k = 0; k < 48; k++) o[k] = w[k];
    hflag[a] = f;
}
__global__ void __launch_bounds__(128) k_sig_prepare(const uint8_t* __restrict__ sig96, uint32_t n, uint32_t* s_aff, uint8_t* sflag) {
    uint32_t a = blockIdx.x * blockDim.x + threadIdx.x;
    if (a >= n) return;
    g2_aff s;
    uint8_t f;
    core_sig_prepare(sig96, a, s, f);
    uint32_t* o = s_aff + 48 * (uint64_t)a;
    const uint32_t* w = reinterpret_cast<const uint32_t*>(&s);
#pragma unroll
    for (int k = 0; k < 48; k++) o[k] = w[k];
    sflag[a] = f;
}
__device__ __forceinline__ g2_aff load_g2_aff(const uint32_t* p) {
    g2_aff r;
    uint32_t* w = reinterpret_cast<uint32_t*>(&r);
#pragma unroll
    for (int k = 0; k < 48; k++) w[k] = p[k];
    return r;
}
// value 2a: miller(PK_agg[a], H(m_a));  value 2a+1: miller(-g1, sig_a).  mode 0: one launch computes both (thread t
// <-> value t); mode 1 / 2: only the pubkey / signature half (thread a), so that the pubkey half can run on a side
// stream while the signatures of the epoch are still being aggregated.
__global__ void __launch_bounds__(128, B2_TAIL_MIN_BLOCKS) k_miller(const uint32_t* __restrict__ pk_jac, const uint8_t* __restrict__ pk_status,
                                                const uint32_t* __restrict__ h_aff, const uint8_t* __restrict__ hflag,
                                                const uint32_t* __restrict__ s_aff, const uint8_t* __restrict__ sflag, uint32_t n_agg,
                                                uint32_t* f_out, int mode, const uint8_t* __restrict__ gpass = nullptr, uint32_t group = 1) {
    uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (mode == 0) {
        if (t >= 2 * n_agg) return;
    } else {
        if (t >= n_agg) return;
        t = 2 * t + (uint32_t)(mode - 1);
    }
    uint32_t a = t >> 1;
    if (gpass && gpass[a / group]) return;      // RLC fallback pass: only the members of a group whose batch equation failed
    fp12 f;
    if (t & 1) {
        f = core_miller_sig(load_g2_aff(s_aff + 48 * (uint64_t)a), sflag[a]);
    } else {
        f = core_miller_pk(pk_jac, pk_status, a, load_g2_aff(h_aff + 48 * (uint64_t)a), hflag[a]);
    }
    uint32_t* o = f_out + 144 * (uint64_t)t;
    const uint32_t* w = reinterpret_cast<const uint32_t*>(&f);
#pragma unroll 1
    for (int k = 0; k < 144; k++) o[k] = w[k];
}
__global__ void __launch_bounds__(128, B2_TAIL_MIN_BLOCKS) k_final_verdict(const uint32_t* __restrict__ f_in, const uint8_t* __restrict__ pk_status,
                                                       const uint8_t* __restrict__ sflag, uint32_t n_agg, uint8_t* ok,
                                                       const uint8_t* __restrict__ gpass = nullptr, uint32_t group = 1) {
    uint32_t a = blockIdx.x * blockDim.x + threadIdx.x;
    if (a >= n_agg) return;
    if (gpass && gpass[a / group]) return;      // RLC fallback pass (see k_miller)
    fp12 f0, f1;
    uint32_t* w0 = reinterpret_cast<uint32_t*>(&f0);
    uint32_t* w1 = reinterpret_cast<uint32_t*>(&f1);
    const uint32_t* p = f_in + 288 * (uint64_t)a;
#pragma unroll 1
    for (int k = 0; k < 144; k++) {
        w0[k] = p[k];
        w1[k] = p[144 + k];
    }
    ok[a] = core_final_verdict(f0, f1, pk_status[a], sflag[a]);
}

// ------------------------------------------------------------------------------------------ bls.SkToPk / bls.Sign (data generation, tests)
__global__ void __launch_bounds__(64) k_sk_to_pk(const uint32_t* __restrict__ sk8, uint64_t n, uint8_t* pk48) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    g1_jac g;
    g.x = fp_load_const(C_G1X);
    g.y = fp_load_const(C_G1Y);
    g.z = fp_one();
    uint32_t k[8];
#pragma unroll
    for (int j = 0; j < 8; j++) k[j] = sk8[8 * i + j];
    g1_compress(pt_mul_var(g, k), pk48 + 48 * i);
}
__global__ void __launch_bounds__(64) k_sign(const uint32_t* __restrict__ sk8, const uint32_t* __restrict__ msg_idx, uint64_t n,
                                              const uint32_t* __restrict__ h_aff, uint8_t* sig96) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    g2_jac h = pt_from_affine(load_g2_aff(h_aff + 48 * (uint64_t)msg_idx[i]));
    uint32_t k[8];
#pragma unroll
    for (int j = 0; j < 8; j++) k[j] = sk8[8 * i + j];
    g2_compress(pt_mul_var(h, k), sig96 + 96 * i);
}
__global__ void __launch_bounds__(64) k_g2_compress_aff(const uint32_t* __restrict__ aff, const uint8_t* __restrict__ inf, uint32_t n, uint8_t* out96) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    g2_compress_affine(load_g2_aff(aff + 48 * (uint64_t)i), inf[i] != 0, out96 + 96 * (uint64_t)i);
}

// ------------------------------------------------------------------------------------------ committee shuffle (SURVEY.md section 8(f)-1)
// compute_shuffled_index (pos-evolution.md:513-534) for every index of the active set at once.
// Stage 1: one thread per hash: source = SHA256(seed || round || LE32(block)) for every 256-index block of every round, and
// pivot = LE64(SHA256(seed || round)[0:8]) mod n per round.  Stage 2: one thread per index walks the rounds in order
// (swap-or-not), reading one source bit per round from the 32 n/256-byte per-round table (L1/L2 resident).
__global__ void __launch_bounds__(128) k_shuffle_sources(const uint8_t* __restrict__ seed32, uint32_t n, uint32_t rounds, uint32_t nblk,
                                                          uint8_t* src, unsigned long long* pivots) {
    // one hash per thread: items 0..nblk-1 of a round are its source blocks, item nblk is its pivot
    uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= rounds * (nblk + 1)) return;
    const uint32_t r = t / (nblk + 1), blk = t % (nblk + 1);
    const bool is_pivot = blk == nblk;
    uint8_t buf[37];
#pragma unroll 1
    for (int i = 0; i < 32; i++) buf[i] = seed32[i];
    buf[32] = (uint8_t)r;
    buf[33] = (uint8_t)blk;
    buf[34] = (uint8_t)(blk >> 8);
    buf[35] = (uint8_t)(blk >> 16);
    buf[36] = (uint8_t)(blk >> 24);
    sha256_ctx c;
    uint8_t out[32];
    sha256_init(c);
    sha256_update(c, buf, is_pivot ? 33u : 37u);
    sha256_final(c, out);
    if (is_pivot) {
        unsigned long long v = 0;
#pragma unroll 1
        for (int i = 7; i >= 0; i--) v = (v << 8) | out[i];
        pivots[r] = v % n;
    } else {
        uint8_t* dst = src + ((uint64_t)r * nblk + blk) * 32;
#pragma unroll 1
        for (int i = 0; i < 32; i++) dst[i] = out[i];
    }
}
// perm[i] = compute_shuffled_index(i); members_out[i] = active[perm[i]] (active == nullptr: identity)
__global__ void __launch_bounds__(256) k_shuffle_apply(uint32_t n, uint32_t rounds, uint32_t nblk, const uint8_t* __restrict__ src,
                                                        const unsigned long long* __restrict__ pivots, const uint32_t* __restrict__ active,
                                                        uint32_t* members_out) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint64_t idx = i;
#pragma unroll 1
    for (uint32_t r = 0; r < rounds; r++) {
        uint64_t flip = (pivots[r] + n - idx) % n;
        uint64_t pos = idx > flip ? idx : flip;
        uint8_t byte = src[((uint64_t)r * nblk + (pos >> 8)) * 32 + ((pos & 255) >> 3)];
        if ((byte >> (pos & 7)) & 1) idx = flip;
    }
    members_out[i] = active ? active[idx] : (uint32_t)idx;
}

// ------------------------------------------------------------------------------------------ K7: update_latest_messages
// Order-exact parallel form of pos-evolution.md:1435-1441.  Table entry = u64 key
// (epoch << 32 | 0xffffffff - order); a stored message has order 0, attestation a of the batch has
// order a+1, so atomicMax picks "highest epoch, earliest in list, stored wins ties" -- exactly the
// sequential rule `i not in latest_messages or target.epoch > latest_messages[i].epoch`.
__device__ __forceinline__ bool lmd_member(const uint32_t* members, const uint32_t* off, const uint8_t* bits, uint32_t stride, uint32_t a,
                                           uint32_t j, uint32_t& v, uint64_t n_val, uint32_t* guard) {
    if (!((bits[(uint64_t)a * stride + (j >> 3)] >> (j & 7)) & 1)) return false;
    v = members[off[a] + j];
    if (v >= n_val) {
        if (guard) atomicOr(guard, (uint32_t)GUARD_BAD_INDEX);
        return false;
    }
    return true;
}
// row size and key of aggregate a for the LMD kernels; false: skip the aggregate (not accepted, malformed row, epoch >= 2^32 - 1)
__device__ __forceinline__ bool lmd_row(const uint32_t* off, uint32_t stride, const uint64_t* target_epoch, const uint8_t* accept, uint32_t a,
                                        uint32_t& size, unsigned long long& key, uint32_t* guard) {
    if (accept && !accept[a]) return false;
    size = guarded_row_size(off, a, stride, guard);
    if (size == 0xffffffffu) return false;
    const unsigned long long e = target_epoch[a];
    if (e >= 0xffffffffull) {                   // would overflow the (epoch << 32 | order) key and break the order-exact election
        if (threadIdx.x == 0 && guard) atomicOr(guard, (uint32_t)GUARD_BAD_EPOCH);
        return false;
    }
    key = (e << 32) | (0xffffffffull - (a + 1));
    return true;
}
__global__ void __launch_bounds__(128) k_lmd_phase1(const uint32_t* __restrict__ members, const uint32_t* __restrict__ off,
                                                     const uint8_t* __restrict__ bits, uint32_t stride, const uint64_t* __restrict__ target_epoch,
                                                     const uint8_t* __restrict__ accept, const uint8_t* __restrict__ equiv, uint32_t n_agg,
                                                     unsigned long long* lmd_key, uint64_t n_val, uint32_t* guard) {
    uint32_t a = blockIdx.x, size, v;
    unsigned long long key;
    if (a >= n_agg || !lmd_row(off, stride, target_epoch, accept, a, size, key, guard)) return;
    for (uint32_t j = threadIdx.x; j < size; j += blockDim.x)
        if (lmd_member(members, off, bits, stride, a, j, v, n_val, guard) && !equiv[v]) atomicMax(&lmd_key[v], key);
}
__global__ void __launch_bounds__(128) k_lmd_phase2(const uint32_t* __restrict__ members, const uint32_t* __restrict__ off,
                                                     const uint8_t* __restrict__ bits, uint32_t stride, const uint64_t* __restrict__ target_epoch,
                                                     const uint32_t* __restrict__ block_idx, const uint8_t* __restrict__ accept,
                                                     const uint8_t* __restrict__ equiv, uint32_t n_agg, unsigned long long* lmd_key,
                                                     uint32_t* lmd_block, uint64_t n_val) {
    uint32_t a = blockIdx.x, size, v;
    unsigned long long key;
    if (a >= n_agg || !lmd_row(off, stride, target_epoch, accept, a, size, key, nullptr)) return;
    for (uint32_t j = threadIdx.x; j < size; j += blockDim.x)
        if (lmd_member(members, off, bits, stride, a, j, v, n_val, nullptr) && !equiv[v] && lmd_key[v] == key) {
            lmd_block[v] = block_idx[a];
            lmd_key[v] = key | 0xffffffffull;
        }
}

// ------------------------------------------------------------------------------------------ K8: vote scatter
// Whether a validator's latest message counts towards get_latest_attesting_balance, in both vote scatters: it exists (key != 0), has not
// expired (key >= min_key, the fork-choice variant's vote expiry), the validator does not equivocate, its flags pass the variant's test
// (flags & flag_mask == flag_need: active, and not slashed when the variant excludes slashed validators), and it names a loaded block.
// The callers have loaded every operand, so the tests are combined without branches.
__device__ __forceinline__ bool latest_message_counts(unsigned long long key, uint32_t block, uint32_t equiv, uint32_t flags, unsigned long long min_key,
                                                      uint32_t flag_need, uint32_t flag_mask, uint32_t n_blocks) {
    return (key != 0) & (key >= min_key) & (equiv == 0) & ((flags & flag_mask) == flag_need) & (block < n_blocks);
}
// One thread per validator: coalesced reads of the latest-message table (u64 key + u32 block), the
// effective-balance table (u64) and two byte masks; votes are combined inside the warp (lanes voting
// for the same block elect a leader) and the leader issues one 64-bit atomic add into the pre-order
// vote array, so that a head everybody agrees on does not serialise a million atomics on one address.
__global__ void __launch_bounds__(256) k_ghost_votes(uint64_t n, const unsigned long long* __restrict__ lmd_key,
                                                      const uint32_t* __restrict__ lmd_block, const uint8_t* __restrict__ equiv,
                                                      const uint8_t* __restrict__ flags, const uint64_t* __restrict__ eff,
                                                      const uint32_t* __restrict__ pre, uint32_t n_blocks, unsigned long long* votes, unsigned long long min_key, uint32_t flag_need, uint32_t flag_mask) {
    uint64_t v = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    bool on = false;
    uint32_t b = 0xffffffffu;
    unsigned long long bal = 0;
    if (v < n) {
        const uint32_t blk = lmd_block[v];
        on = latest_message_counts(lmd_key[v], blk, equiv[v], flags[v], min_key, flag_need, flag_mask, n_blocks);
        if (on) {
            b = pre[blk];
            bal = eff[v];
        }
    }
    const int lane = threadIdx.x & 31;
    unsigned peers = __match_any_sync(B2_FULL_MASK, b);
    unsigned long long sum = 0;
#pragma unroll
    for (int l = 0; l < 32; l++) {
        unsigned long long o = __shfl_sync(B2_FULL_MASK, bal, l);
        if ((peers >> l) & 1u) sum += o;
    }
    if (on && lane == __ffs(peers) - 1) atomicAdd(&votes[b], sum);
}

// The validators [v_begin, v_end) of a vote scatter: their latest-message, equivocation, flag and balance tables offset to v_begin
// (n = v_end - v_begin), and the fork-choice variant (votes below min_key expire; flags & flag_mask must equal flag_need)
struct ghost_votes_args {
    uint64_t n;
    const unsigned long long* lmd_key;
    const uint32_t* lmd_block;
    const uint8_t *equiv, *flags;
    const uint64_t* eff;
    unsigned long long min_key;
    uint32_t flag_need, flag_mask;
};
// Same scatter with the per-block bins privatised in shared memory (used when n_blocks * 8 B fits): a persistent grid
// of one CTA per SM strides over the validators; lanes of a warp voting for the same block are combined first, the
// leader adds into the CTA's shared bins, and only non-zero bins are flushed to global memory -- one atomic per
// (CTA, voted block) instead of one per (warp, voted block), which matters when a million validators agree on a
// handful of recent blocks (the realistic case) and the global atomics would serialise on those addresses.
__device__ __forceinline__ void ghost_votes_body(unsigned long long* bins, const ghost_votes_args& V, const uint32_t* __restrict__ pre, uint32_t n_blocks,
                                                 unsigned long long* votes, unsigned long long* dbg = nullptr) {
#define B2_VOTE_STAMP(k) do { if (dbg && blockIdx.x == 0 && threadIdx.x == 0) dbg[k] = clock64(); } while (0)
    B2_VOTE_STAMP(16);
    for (uint32_t i = threadIdx.x; i < n_blocks; i += blockDim.x) bins[i] = 0;
    __syncthreads();
    B2_VOTE_STAMP(17);
    const int lane = threadIdx.x & 31;
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    const uint64_t n_round = (V.n + stride - 1) / stride * stride;          // whole warps stay converged for the shuffles
    // Four validators per thread and trip: all twenty table loads (key, block, balance, flags, equivocation byte -- addresses depend on
    // the validator index only) are issued before the first is used, then the one dependent gather (block -> pre-order position, a
    // 40 KB table that lives in L1).  The round-1 form tested `key != 0 && ...` load by load, i.e. four dependent round trips per
    // validator (ncu: 72 % of the samples in stall_long_sb at those four points, on an earlier GPU).
    constexpr int U = 4;
    for (uint64_t v0 = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; v0 < n_round; v0 += U * stride) {
        unsigned long long key[U], bal[U];
        uint32_t blk[U], fl[U], eq[U];
#pragma unroll
        for (int u = 0; u < U; u++) {
            const uint64_t v = v0 + u * stride;
            const bool in = v < V.n;
            key[u] = in ? V.lmd_key[v] : 0ull;
            blk[u] = in ? V.lmd_block[v] : 0u;
            bal[u] = in ? V.eff[v] : 0ull;
            fl[u] = in ? V.flags[v] : 0u;
            eq[u] = in ? V.equiv[v] : 1u;
        }
        uint32_t b[U];
        bool on[U];
#pragma unroll
        for (int u = 0; u < U; u++) {
            on[u] = latest_message_counts(key[u], blk[u], eq[u], fl[u], V.min_key, V.flag_need, V.flag_mask, n_blocks);
            b[u] = on[u] ? pre[blk[u]] : 0xffffffffu;
        }
#pragma unroll
        for (int u = 0; u < U; u++) {
            if (v0 + u * stride >= n_round) break;                          // warp-uniform
            // fast path: the whole warp votes for one block (the common case on a healthy chain): one shuffle reduction, one
            // shared-memory atomic.  Otherwise every lane adds into the CTA-private bins itself (shared-memory atomics).
            const unsigned voting = __ballot_sync(B2_FULL_MASK, on[u]);
            if (voting == 0) continue;
            const uint32_t b0 = __shfl_sync(B2_FULL_MASK, b[u], __ffs(voting) - 1);
            const bool uniform = __all_sync(B2_FULL_MASK, !on[u] || b[u] == b0);
            if (uniform) {
                unsigned long long sum = on[u] ? bal[u] : 0ull;
#pragma unroll
                for (int d = 16; d >= 1; d >>= 1) sum += __shfl_down_sync(B2_FULL_MASK, sum, d);
                if (lane == 0) atomicAdd(&bins[b0], sum);
            } else if (on[u]) {
                atomicAdd(&bins[b[u]], bal[u]);
            }
        }
    }
    __syncthreads();
    B2_VOTE_STAMP(18);
    for (uint32_t i = threadIdx.x; i < n_blocks; i += blockDim.x) {
        unsigned long long w = bins[i];
        if (w) atomicAdd(&votes[i], w);
    }
    B2_VOTE_STAMP(19);
}
// The two scatter kernels take the tables as separate __restrict__ parameters rather than a ghost_votes_args: only a restrict-qualified
// kernel parameter lets the compiler read them through the read-only path (LDG.CONSTANT).
__global__ void __launch_bounds__(1024) k_ghost_votes_smem(uint64_t n, const unsigned long long* __restrict__ lmd_key,
                                                            const uint32_t* __restrict__ lmd_block, const uint8_t* __restrict__ equiv,
                                                            const uint8_t* __restrict__ flags, const uint64_t* __restrict__ eff,
                                                            const uint32_t* __restrict__ pre, uint32_t n_blocks, unsigned long long* votes, unsigned long long min_key, uint32_t flag_need, uint32_t flag_mask) {
    extern __shared__ unsigned long long bins[];
    ghost_votes_body(bins, ghost_votes_args{n, lmd_key, lmd_block, equiv, flags, eff, min_key, flag_need, flag_mask}, pre, n_blocks, votes);
}

// ------------------------------------------------------------------------------------------ K9: subtree weights + head
// Single block.  b2_tree_load renumbers the blocks in DFS pre-order and stores every per-block array in that order, so
//   * the subtree of the block at position p is the contiguous range [p, p + size[p]) and its
//     get_latest_attesting_balance is a difference of two prefix sums of the direct votes (+ boost on one block);
//   * the children of p are p+1, p+1+size[p+1], ... -- no child lists;
//   * all loads are coalesced and everything lives in shared memory (16 B per block).
// The head walk of get_head (argmax over children of (weight, root), repeated down to a leaf) needs no pointer chasing:
// mark every block that is NOT the best child of its parent; a block lies on the head path iff no block on its root path is
// marked, i.e. iff the number of marked ancestors-or-self is zero.  That count is a second prefix sum (+1 at the marked block,
// -1 past its subtree), and the head is the last pre-order position with count zero -- two scans and a max-reduction
// instead of log2(n) rounds over all blocks.  Trees too large for shared memory run the same algorithm on global memory (the generic
// form, ghost_tree_body).  b2_tree_load chooses the form and builds only the tables it reads; the others are null.
struct ghost_tree_args {
    uint32_t n;
    const uint32_t* pre;         // block -> pre-order position
    const uint32_t* inv;         // pre-order position -> block
    const uint32_t* size_keep;   // generic form, pre-order: subtree size | (get_filtered_block_tree membership << 31)
    const uint32_t* rank;        // generic form, pre-order: lexicographic rank of the 32-byte root (tie-break of :1114-1116)
    const uint32_t* packed;      // shared-memory form, pre-order: size | rank << 15 | keep << 31 (one word per block)
    unsigned long long* votes;   // in: direct votes in pre-order; zeroed on exit
    unsigned long long* g_w;     // generic form scratch n+1 (prefix sums)
    unsigned long long* g_w2;    // generic form scratch n (weights)
    uint32_t* g_next;            // generic form scratch n+1 (marks / counts)
    unsigned long long* weight_out;  // optional, per block (original numbering)
    uint32_t* head_out;
    uint32_t* host_out;          // optional: mapped pinned host memory that receives (head, host_seq) in one 64-bit store
    uint32_t host_seq;
    uint32_t justified;
    int32_t boost_idx;
    unsigned long long boost_score;
    int use_smem;                // the shared-memory form (ghost_tree_smem) on packed; else the generic form
    int hard_list;               // shared-memory form: the launch reserved u32[n] more for the work list of the marking phase
    unsigned long long* dbg;     // optional: thread 0 of the tree phase stores clock64() at its phase boundaries (b2_debug_head_clocks)
};
#define B2_TREE_STAMP(k) do { if (A.dbg && threadIdx.x == 0) A.dbg[k] = clock64(); } while (0)

// exclusive prefix sum of x[0..n) in place, x[n] = total; every thread of the block must call it
template <class T> __device__ __forceinline__ void block_exclusive_scan(T* x, uint32_t n, T* warp_tot) {
    const uint32_t tid = threadIdx.x, nthr = blockDim.x;
    const uint32_t per = (n + nthr - 1) / nthr;
    const uint32_t lo = min(n, tid * per), hi = min(n, lo + per);
    T local = 0;
    for (uint32_t i = lo; i < hi; i++) local += x[i];
    T incl = local;
    const int lane = tid & 31, warp = tid >> 5;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        T o = __shfl_up_sync(B2_FULL_MASK, incl, d);
        if (lane >= d) incl += o;
    }
    if (lane == 31) warp_tot[warp] = incl;
    __syncthreads();
    if (warp == 0) {
        T w = (lane < (int)(nthr >> 5)) ? warp_tot[lane] : 0, wi = w;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            T o = __shfl_up_sync(B2_FULL_MASK, wi, d);
            if (lane >= d) wi += o;
        }
        warp_tot[lane] = wi - w;
    }
    __syncthreads();
    T run = warp_tot[warp] + incl - local;
    for (uint32_t i = lo; i < hi; i++) {
        T v = x[i];
        x[i] = run;
        run += v;
    }
    if (lo < n && hi == n) x[n] = run;
    if (n == 0 && tid == 0) x[0] = 0;
    __syncthreads();
}

// get_weight of every block, in the original numbering, from the weights w[] in pre-order
__device__ __forceinline__ void store_weights(const ghost_tree_args& A, const unsigned long long* w) {
    if (A.weight_out)
        for (uint32_t b = threadIdx.x; b < A.n; b += blockDim.x) A.weight_out[b] = w[A.pre[b]];
}
// The end of the tree phase in both forms.  After the second scan mark[p+1] is the inclusive count at p = number of marked blocks among
// p and its ancestors.  The head path below the justified block (at pre-order position jp) = the positions of its subtree whose count
// equals the justified block's own count (nothing marked in between); the head is the last of them in pre-order.  The subtree sizes are
// the size_mask bits of the form's per-block words size[].  Thread 0 stores the head to A.head_out and, if A.host_out is set, publishes
// it there with A.host_seq.
__device__ __forceinline__ void ghost_tree_head(const ghost_tree_args& A, const uint32_t* mark, const uint32_t* size, uint32_t size_mask, uint32_t jp,
                                                uint32_t& head_pos) {
    const uint32_t base = mark[jp + 1];
    const uint32_t jend = jp + (size[jp] & size_mask);
    uint32_t best_pos = 0;
    bool have = false;
    for (uint32_t p = jp + threadIdx.x; p < jend; p += blockDim.x) {
        if (mark[p + 1] == base) {
            best_pos = p;
            have = true;
        }
    }
    if (have) atomicMax(&head_pos, best_pos);
    __syncthreads();
    B2_TREE_STAMP(7);
    if (threadIdx.x == 0) {
        const uint32_t h = (A.justified < A.n) ? A.inv[max(head_pos, jp)] : 0xffffffffu;
        *A.head_out = h;
        if (A.host_out)                         // zero-copy result: (head, sequence number) in one 64-bit store to mapped pinned memory
            *reinterpret_cast<volatile unsigned long long*>(A.host_out) = (unsigned long long)h | ((unsigned long long)A.host_seq << 32);
    }
    B2_TREE_STAMP(15);
}

// The generic form of the tree phase, for trees too large for shared memory: the tables and scratch of b2_tree_load in global memory.
__device__ __forceinline__ void ghost_tree_body(const ghost_tree_args& A) {
    __shared__ unsigned long long warp_tot[32];
    __shared__ uint32_t warp_tot32[32];
    __shared__ uint32_t head_pos;
    const uint32_t n = A.n, tid = threadIdx.x, T = blockDim.x;
    B2_TREE_STAMP(0);
    unsigned long long* W = A.g_w;                                          // n+1: votes -> prefix sums
    const uint32_t* size = A.size_keep;                                     // n
    uint32_t* mark = A.g_next;                                              // n+1: marks -> counts
    const uint32_t boost_p = A.boost_idx >= 0 ? A.pre[A.boost_idx] : 0xffffffffu;
    if (tid == 0) head_pos = 0;
    // stage votes (+ boost), coalesced; leave the global accumulator clean for the next call
    for (uint32_t p = tid; p < n; p += T) {
        unsigned long long v = __ldcg(&A.votes[p]);
        A.votes[p] = 0;
        if (p == boost_p) v += A.boost_score;
        W[p] = v;
        mark[p] = 0;
    }
    if (tid == 0) mark[n] = 0;
    __syncthreads();
    B2_TREE_STAMP(1);
    block_exclusive_scan(W, n, warp_tot);
    B2_TREE_STAMP(2);
    // weights: w[p] = S[p + size] - S[p]
    unsigned long long* Wt = A.g_w2;
    for (uint32_t p = tid; p < n; p += T) Wt[p] = W[p + (size[p] & 0x7fffffffu)] - W[p];
    __syncthreads();
    B2_TREE_STAMP(4);
    store_weights(A, Wt);
    // every child that is not its parent's best child gets +1 at its position and -1 just past its subtree
    const uint32_t jp = A.justified < n ? A.pre[A.justified] : 0;
    for (uint32_t p = tid; p < n; p += T) {
        const uint32_t sk = size[p];
        const uint32_t end = p + (sk & 0x7fffffffu);
        if (p + 1 >= end) continue;
        uint32_t best = 0xffffffffu;
        if (sk >> 31) {
            unsigned long long bw = 0;
            for (uint32_t c = p + 1; c < end; c += size[c] & 0x7fffffffu) {
                if (!(size[c] >> 31)) continue;
                const unsigned long long w = Wt[c];
                if (best == 0xffffffffu || w > bw || (w == bw && A.rank[c] > A.rank[best])) {
                    best = c;
                    bw = w;
                }
            }
        }
        for (uint32_t c = p + 1; c < end; c += size[c] & 0x7fffffffu)
            if (c != best) {
                atomicAdd(&mark[c], 1u);
                atomicAdd(&mark[c + (size[c] & 0x7fffffffu)], 0xffffffffu);     // -1 (mod 2^32); position n is the sentinel slot
            }
    }
    __syncthreads();
    B2_TREE_STAMP(5);
    block_exclusive_scan(mark, n, warp_tot32);          // mark[p] = number of marked proper ancestors ... of positions < p
    B2_TREE_STAMP(6);
    ghost_tree_head(A, mark, size, 0x7fffffffu, jp, head_pos);
}
// ---- the shared-memory form of the tree phase (every tree that fits: <= 14 463 blocks), specialised after the phase clocks of the
// generic body run on shared memory (tools/head_clocks.py on an earlier GPU: 44 900 SM clocks = 23.6 us, of which marking 17 800, staging 8 700, first scan
// 6 100): (1) all arrays are __shared__ pointers -- LDS/STS instead of generic LD/ST whose address space is resolved at run time;
// (2) the per-block word packs subtree size, root rank and the filter bit, so a tie between equal-weight siblings costs no global
// load (the generic body reads A.rank[] from global memory inside the child loop); (3) the staging loop issues all of a thread's
// global loads before using any; (4) the prefix sums are raking scans (registers, one warp scan per warp, one cross-warp
// step); (5) the head and its sequence number leave in ONE 64-bit store to mapped host memory.
#define B2_SZ(x) ((x) & 0x7fffu)
#define B2_RK(x) (((x) >> 15) & 0x7fffu)
#define B2_KEEP(x) ((x) >> 31)
// exclusive prefix sum of x[0..n) in shared memory, x[n] = total.  Raking form: thread t owns the K consecutive elements from t*K
// (K = ceil(n / threads) made odd, so the thread stride is conflict-free for 32- and 64-bit words alike), sums them in registers, the
// block scans the 1 024 thread totals with one warp scan per warp plus one over the 32 warp totals, and every thread writes its
// running prefix back: one load pass, one store pass, 5 shuffle steps per WARP.  The row-wise form it replaces (a 5-step shuffle scan
// per ROW of 32, 313 rows) sat on the block's one shuffle unit: 6 200 clocks for the u64 scan and 3 500 for the u32 one
// (tools/head_clocks.py).
template <class T, int MAXPT> __device__ __forceinline__ void smem_exclusive_scan(T* x, uint32_t n, T* warp_tot) {
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nwarp = blockDim.x >> 5;
    const uint32_t K = ((n + blockDim.x - 1) / blockDim.x) | 1u;           // <= MAXPT: the caller's n <= MAXPT * threads, MAXPT odd
    const uint32_t i0 = tid * K;
    T v[MAXPT];
    T tot = 0;
#pragma unroll
    for (int j = 0; j < MAXPT; j++) {
        const uint32_t i = i0 + j;
        v[j] = ((uint32_t)j < K && i < n) ? x[i] : (T)0;
        tot += v[j];
    }
    T incl = tot;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const T o = __shfl_up_sync(B2_FULL_MASK, incl, d);
        if ((int)lane >= d) incl += o;
    }
    if (lane == 31) warp_tot[warp] = incl;
    __syncthreads();
    if (warp == 0) {
        const T w = lane < nwarp ? warp_tot[lane] : (T)0;
        T wi = w;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const T o = __shfl_up_sync(B2_FULL_MASK, wi, d);
            if ((int)lane >= d) wi += o;
        }
        warp_tot[lane] = wi - w;                                            // exclusive offset of each warp
        if (lane == 31) x[n] = wi;                                          // grand total
    }
    __syncthreads();
    T run = warp_tot[warp] + incl - tot;                                    // exclusive prefix of the thread's first element
#pragma unroll
    for (int j = 0; j < MAXPT; j++) {
        const uint32_t i = i0 + j;
        if ((uint32_t)j < K && i < n) x[i] = run;
        run += v[j];
    }
    __syncthreads();
}
// MAXPT = elements per thread the unrolled loops are built for (odd, n <= MAXPT * 1024).  The block's 32 warps share four issue
// slots, so the phase times are instruction counts: the 15-trip form spends a third of its instructions on predicated-off trips
// when n = 10 000 needs 10 (11 in the scans), hence the two instantiations behind ghost_tree_smem().
template <int MAXPT>
__device__ __forceinline__ void ghost_tree_smem_t(const ghost_tree_args& A, unsigned long long* smem_u64, unsigned long long* warp_tot, uint32_t* warp_tot32,
                                                  uint32_t* cells) {
    uint32_t& head_pos = cells[0];
    uint32_t& n_hard = cells[1];
    const uint32_t n = A.n, tid = threadIdx.x, T = blockDim.x;
    B2_TREE_STAMP(0);
    unsigned long long* W = smem_u64;                                       // n+1: votes -> prefix sums -> weights
    uint32_t* sz = reinterpret_cast<uint32_t*>(smem_u64 + (n + 1));         // n: size | rank << 15 | keep << 31
    uint32_t* mark = sz + n;                                                // n+1: marks -> counts
    const uint32_t boost_p = A.boost_idx >= 0 ? __ldg(A.pre + A.boost_idx) : 0xffffffffu;
    const uint32_t jp = A.justified < n ? __ldg(A.pre + A.justified) : 0;
    if (tid == 0) head_pos = 0;
    {
        unsigned long long v[MAXPT];
        uint32_t s[MAXPT];
#pragma unroll
        for (int j = 0; j < MAXPT; j++) {                                   // every global load of the thread in flight at once
            const uint32_t p = tid + j * T;
            v[j] = p < n ? __ldcg(A.votes + p) : 0ull;
            s[j] = p < n ? __ldg(A.packed + p) : 0u;
        }
#pragma unroll
        for (int j = 0; j < MAXPT; j++) {
            const uint32_t p = tid + j * T;
            if (p < n) {
                A.votes[p] = 0;                                             // leave the global accumulator clean for the next call
                W[p] = v[j] + (p == boost_p ? A.boost_score : 0ull);
                sz[p] = s[j];
                mark[p] = 0;
            }
        }
    }
    if (tid == 0) mark[n] = 0;
    __syncthreads();
    B2_TREE_STAMP(1);
    smem_exclusive_scan<unsigned long long, MAXPT>(W, n, warp_tot);
    B2_TREE_STAMP(2);
    {
        unsigned long long wreg[MAXPT];
#pragma unroll
        for (int j = 0; j < MAXPT; j++) {
            const uint32_t p = tid + j * T;
            if (p < n) wreg[j] = W[p + B2_SZ(sz[p])] - W[p];                 // weight = difference of two prefix sums
        }
        __syncthreads();
        B2_TREE_STAMP(3);
#pragma unroll
        for (int j = 0; j < MAXPT; j++) {
            const uint32_t p = tid + j * T;
            if (p < n) W[p] = wreg[j];
        }
    }
    __syncthreads();
    B2_TREE_STAMP(4);
    store_weights(A, W);
    // every child that is not its parent's best child gets +1 at its position and -1 just past its subtree.
    // Most parents of a block tree have ONE child (the chain); it is trivially the best child and nothing is marked.  Looping over
    // parents thread by thread makes every warp wait for its lane with the most children in each of its ~10 trips (13 800 clocks).
    // When the launch left room for a work list (A.hard_list), the parents that need the loops are first compacted into it and
    // then spread evenly over the block.
    // One traversal per parent (the child chain c -> c + size[c] is a chain of dependent shared-memory loads): every child is marked as
    // it is visited, the best one is remembered and un-marked at the end -- two more shared atomics per parent instead of a second walk.
    auto mark_children = [&](uint32_t p, uint32_t sk) {
        const uint32_t end = p + B2_SZ(sk);
        const bool pick = B2_KEEP(sk) != 0;             // a block outside the filtered tree has no best child
        uint32_t best = 0xffffffffu, best_rk = 0, best_step = 0;
        unsigned long long bw = 0;
        for (uint32_t c = p + 1; c < end;) {
            const uint32_t sc = sz[c];
            const uint32_t step = B2_SZ(sc);
            atomicAdd(&mark[c], 1u);
            atomicAdd(&mark[c + step], 0xffffffffu);                        // -1 (mod 2^32); position n is the sentinel slot
            if (pick && B2_KEEP(sc)) {
                const unsigned long long w = W[c];
                if (best == 0xffffffffu || w > bw || (w == bw && B2_RK(sc) > best_rk)) {
                    best = c;
                    bw = w;
                    best_rk = B2_RK(sc);
                    best_step = step;
                }
            }
            c += step;
        }
        if (best != 0xffffffffu) {
            atomicAdd(&mark[best], 0xffffffffu);
            atomicAdd(&mark[best + best_step], 1u);
        }
    };
    if (A.hard_list) {
        uint32_t* list = mark + (n + 1);                                    // u32[n], behind the three arrays
        if (tid == 0) n_hard = 0;
        __syncthreads();
        const uint32_t lane = tid & 31;
        // all of a thread's tests first (their loads overlap), ONE reservation per warp: a reservation per trip was 320 returning
        // atomics on one shared word, each trip waiting for its own
        unsigned hm[MAXPT];
        uint32_t wcount = 0;
#pragma unroll
        for (int j = 0; j < MAXPT; j++) {
            const uint32_t p = tid + j * T;
            bool hard = false;
            if (p < n) {
                const uint32_t sk = sz[p];
                if (B2_SZ(sk) > 1) {
                    const uint32_t s1 = sz[p + 1];                          // p has a child, so p + 1 < n
                    hard = !(B2_SZ(s1) + 1 == B2_SZ(sk) && B2_KEEP(sk) && B2_KEEP(s1));      // not "one child, kept": needs the loops
                }
            }
            hm[j] = __ballot_sync(B2_FULL_MASK, hard);
            wcount += __popc(hm[j]);
        }
        uint32_t at = 0;
        if (lane == 0 && wcount) at = atomicAdd(&n_hard, wcount);
        at = __shfl_sync(B2_FULL_MASK, at, 0);
#pragma unroll
        for (int j = 0; j < MAXPT; j++) {
            if ((hm[j] >> lane) & 1u) list[at + __popc(hm[j] & ((1u << lane) - 1u))] = tid + j * T;
            at += __popc(hm[j]);
        }
        __syncthreads();
        B2_TREE_STAMP(8);
        const uint32_t nh = n_hard;
        for (uint32_t i = tid; i < nh; i += T) {
            const uint32_t p = list[i];
            mark_children(p, sz[p]);
        }
    } else {
        for (uint32_t p = tid; p < n; p += T) {
            const uint32_t sk = sz[p];
            if (B2_SZ(sk) > 1) mark_children(p, sk);
        }
    }
    __syncthreads();
    B2_TREE_STAMP(5);
    smem_exclusive_scan<uint32_t, MAXPT>(mark, n, warp_tot32);
    B2_TREE_STAMP(6);
    ghost_tree_head(A, mark, sz, 0x7fffu, jp, head_pos);             // the B2_SZ field
}
__device__ __forceinline__ void ghost_tree_smem(const ghost_tree_args& A, unsigned long long* smem_u64) {
    __shared__ unsigned long long warp_tot[32];
    __shared__ uint32_t warp_tot32[32];
    __shared__ uint32_t cells[2];                                           // head position, length of the work list
    if (A.n <= 11u * blockDim.x) ghost_tree_smem_t<11>(A, smem_u64, warp_tot, warp_tot32, cells);
    else ghost_tree_smem_t<15>(A, smem_u64, warp_tot, warp_tot32, cells);      // n <= 15 * 1024: tree_form_of's smem_tree test
}

__global__ void __launch_bounds__(1024) k_ghost_tree(ghost_tree_args A) {
    extern __shared__ unsigned long long smem_u64[];
    if (A.use_smem)
        ghost_tree_smem(A, smem_u64);
    else
        ghost_tree_body(A);
}
// get_head in ONE launch (b2_get_head): every CTA scatters its share of the votes (K8), the CTA that finishes last -- elected by a
// ticket counter -- runs the tree phase (K9) on the completed vote array and writes the head straight into mapped pinned host memory
// (head, then a sequence number the host spins on): no second launch, no device-to-host copy, no stream synchronisation.
// Called by every thread after its CTA's scatter: true in the CTA whose ticket completes the grid, which re-arms the ticket for the
// next call.  `is_last` is a __shared__ flag of the calling kernel (declared there, the kernel keeps its shared-memory layout).
__device__ __forceinline__ bool last_cta(unsigned int* ticket, bool& is_last) {
    __syncthreads();                                   // every flush atomic of this CTA has been issued
    if (threadIdx.x == 0) {
        __threadfence();
        is_last = atomicAdd(ticket, 1u) == gridDim.x - 1;
    }
    __syncthreads();
    if (!is_last) return false;
    __threadfence();                                   // the other CTAs' vote atomics are visible (they live in L2)
    if (threadIdx.x == 0) *ticket = 0;                 // re-armed for the next call
    return true;
}
__global__ void __launch_bounds__(1024) k_get_head_fused(ghost_votes_args V, ghost_tree_args A, unsigned int* ticket) {
    extern __shared__ unsigned long long smem_u64[];
    __shared__ bool is_last;
    ghost_votes_body(smem_u64, V, A.pre, A.n, A.votes, A.dbg);
    if (!last_cta(ticket, is_last)) return;
    ghost_tree_smem(A, smem_u64);                      // (the fused kernel is only launched for trees in the shared-memory form)
}

// get_head over ONE validator set spread over the GPUs of a box (BASELINE.json config 4: N/8 validators per GPU) as one kernel per rank,
// the all-reduce of the per-block vote weights fused into it over NVLink peer memory:
//   1. every CTA scatters its share of THIS RANK's validators into the rank's local vote vector (as k_get_head_fused);
//   2. the CTA that finishes last PUSHES the rank's vector into the accumulator of every rank of the box -- 64-bit reductions
//      (red.add) straight into peer memory mapped through CUDA IPC, 80 KB per peer through NVSwitch -- then raises its flag on every
//      peer (system-scope release) and waits until every rank's flag for this call has arrived in its own flag row;
//   3. it then runs the tree phase on the now complete accumulator and publishes the head (zero-copy).
// No NCCL launch, no second kernel, no host round trip between the stages.  Calls are collective: every rank must issue them in the
// same order (the sequence number).  Accumulators and flag rows are double-buffered by the parity of the sequence number, so a rank
// that races ahead into call k+1 never touches the buffers call k is still reading.
#define B2_MAX_PEERS 8
struct ghost_peer_args {
    unsigned long long* acc[B2_MAX_PEERS];     // acc[r]: rank r's accumulators, 2 x n_blocks u64 (parity-major), peer-mapped
    unsigned int* flags[B2_MAX_PEERS];         // flags[r]: rank r's flag rows, 2 x B2_MAX_PEERS u32
    uint32_t rank, world, seq;
};
__global__ void __launch_bounds__(1024) k_get_head_fused_nvl(ghost_votes_args V, ghost_tree_args A, ghost_peer_args P, unsigned int* ticket,
                                                              unsigned long long* local_votes) {
    extern __shared__ unsigned long long smem_u64[];
    __shared__ bool is_last;
    ghost_votes_body(smem_u64, V, A.pre, A.n, local_votes, A.dbg);
    if (!last_cta(ticket, is_last)) return;
    const uint32_t par = P.seq & 1u, n = A.n;
    // push: this rank's direct votes into every rank's accumulator (own included); the local vector is left clean for the next call
    for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) {
        const unsigned long long w = __ldcg(local_votes + i);
        if (w) {
            local_votes[i] = 0;
            for (uint32_t r = 0; r < P.world; r++) atomicAdd(P.acc[r] + (size_t)par * n + i, w);      // RED.ADD.64 over NVLink for r != rank
        }
    }
    __threadfence_system();
    __syncthreads();
    if (threadIdx.x < P.world) {
        // raise my flag on rank `threadIdx.x`, then wait for that rank's flag in my own row
        volatile unsigned int* theirs = P.flags[threadIdx.x] + par * B2_MAX_PEERS + P.rank;
        *theirs = P.seq;
        volatile unsigned int* mine = P.flags[P.rank] + par * B2_MAX_PEERS + threadIdx.x;
        while (*mine != P.seq) {
        }
    }
    __threadfence_system();
    __syncthreads();
    A.votes = P.acc[P.rank] + (size_t)par * n;         // the tree phase reads (ld.cg) and zeroes the complete accumulator
    ghost_tree_smem(A, smem_u64);
}

}  // namespace b2

// ------------------------------------------------------------------------------------------ K5/K6, 3-lane team versions
#include "team.cuh"
namespace b2 {

#define B2_TEAMS_PER_WARP 10         // 30 of 32 lanes; 10 * sizeof(team_ws) = 48 960 B of shared memory per (one-warp) block

// value index `item`: mode 0: item in [0, 2n): even = pubkey half, odd = signature half; mode 1/2: item = aggregate
__global__ void __launch_bounds__(32) k_miller_team(const uint32_t* __restrict__ pk_jac, const uint8_t* __restrict__ pk_status,
                                                     const uint32_t* __restrict__ h_aff, const uint8_t* __restrict__ hflag,
                                                     const uint32_t* __restrict__ s_aff, const uint8_t* __restrict__ sflag, uint32_t n_agg,
                                                     uint32_t* f_out, int mode) {
    extern __shared__ unsigned long long team_smem[];
    team_ws* wsv = reinterpret_cast<team_ws*>(team_smem);
    const int lane = threadIdx.x, tt = lane / 3, l = lane % 3;
    const uint32_t n_items = mode == 0 ? 2 * n_agg : n_agg;
    uint32_t item = blockIdx.x * B2_TEAMS_PER_WARP + tt;
    if (tt >= B2_TEAMS_PER_WARP || item >= n_items) return;
    uint32_t t = mode == 0 ? item : 2 * item + (uint32_t)(mode - 1);
    const uint32_t a = t >> 1;
    team tm = {l, 7u << (3 * tt), nullptr};
    team_ws* ws = wsv + tt;
    if (t & 1) {
        const uint8_t sf = sflag[a];
        if (sf == SIG_INVALID) {
            if (l == 0) ws->f = fp12_one();
            team_sync(tm);
        } else {
            g1_jac ng;
            ng.x = fp_load_const(C_G1X);
            ng.y = fp_load_const(C_G1Y_NEG);
            ng.z = fp_one();
            team_miller_loop(tm, ws, ng, load_g2_aff(s_aff + 48 * (uint64_t)a), sf == SIG_INFINITY);
        }
    } else {
        if (pk_status[a] != PK_OK) {
            if (l == 0) ws->f = fp12_one();
            team_sync(tm);
        } else {
            team_miller_loop(tm, ws, load_g1_jac(pk_jac + 36 * (uint64_t)a), load_g2_aff(h_aff + 48 * (uint64_t)a), hflag[a] != 0);
        }
    }
    uint32_t* o = f_out + 144 * (uint64_t)t;
    const uint32_t* w = reinterpret_cast<const uint32_t*>(&ws->f);
#pragma unroll 1
    for (int k = l; k < 144; k += 3) o[k] = w[k];
}

__global__ void __launch_bounds__(32) k_final_team(const uint32_t* __restrict__ f_in, const uint8_t* __restrict__ pk_status,
                                                    const uint8_t* __restrict__ sflag, uint32_t n_agg, uint8_t* ok) {
    extern __shared__ unsigned long long team_smem[];
    team_ws* wsv = reinterpret_cast<team_ws*>(team_smem);
    const int lane = threadIdx.x, tt = lane / 3, l = lane % 3;
    const uint32_t a = blockIdx.x * B2_TEAMS_PER_WARP + tt;
    if (tt >= B2_TEAMS_PER_WARP || a >= n_agg) return;
    team tm = {l, 7u << (3 * tt), nullptr};
    team_ws* ws = wsv + tt;
    if (pk_status[a] != PK_OK || sflag[a] == SIG_INVALID) {
        if (l == 0) ok[a] = 0;
        return;
    }
    const uint32_t* p = f_in + 288 * (uint64_t)a;
    uint32_t* w0 = reinterpret_cast<uint32_t*>(&ws->g);
    uint32_t* w1 = reinterpret_cast<uint32_t*>(&ws->h);
#pragma unroll 1
    for (int k = l; k < 144; k += 3) {
        w0[k] = p[k];
        w1[k] = p[144 + k];
    }
    team_sync(tm);
    team_fp12_mul(tm, ws, &ws->f, &ws->g, &ws->h);
    team_final_exponentiation(tm, ws);
    if (l == 0) ok[a] = fp12_is_one(ws->f) ? 1 : 0;
}

}  // namespace b2

// ------------------------------------------------------------------------------------------ batched SHA-256 (fixed-length messages)
// `hash` of the spec (pos-evolution.md:486, :522, :525): n messages of msg_len bytes each -> n digests.  Building block of
// the committee shuffle and of device-side SSZ merkleization (SURVEY.md section 8(f)-3).
namespace b2 {
__global__ void __launch_bounds__(128) k_sha256_fixed(const uint8_t* __restrict__ in, uint32_t msg_len, uint64_t n, uint8_t* out) {
    uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    sha256_ctx c;
    uint8_t d[32];
    sha256_init(c);
    sha256_update(c, in + i * msg_len, msg_len);
    sha256_final(c, d);
#pragma unroll 1
    for (int k = 0; k < 32; k++) out[32 * i + k] = d[k];
}
}  // namespace b2
static_assert(B2_TEAMS_PER_WARP * 3 <= 32, "a warp holds at most 10 three-lane teams");
static_assert(B2_TEAMS_PER_WARP * sizeof(b2::team_ws) <= 48 * 1024, "team workspaces must fit the default dynamic shared memory limit");

// ------------------------------------------------------------------------------------------ SSZ signing roots on the device (SURVEY.md section 8(f)-3)
// compute_signing_root(AttestationData, domain) (pattern of pos-evolution.md:163; containers :689-697, :219-221):
//   hash_tree_root(AttestationData) = Merkle root of 8 chunks [slot, index, beacon_block_root, htr(source), htr(target), 0, 0, 0],
//   htr(Checkpoint) = SHA256(pad32(LE64(epoch)) || root), signing root = SHA256(object_root || domain).
// Input record = the 128-byte SSZ serialisation of AttestationData (slot u64, index u64, beacon_block_root, source.epoch u64,
// source.root, target.epoch u64, target.root).  One thread per attestation, 10 two-block SHA-256 evaluations.
namespace b2 {
// domain_stride = 0: one domain for the whole batch; 32: one per attestation
__global__ void __launch_bounds__(64) k_signing_roots(const uint8_t* __restrict__ data128, const uint8_t* __restrict__ domain32, uint32_t domain_stride,
                                                       uint32_t n, uint8_t* out32) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint8_t d[128], dom[32], o[32];
    for (int k = 0; k < 128; k++) d[k] = data128[128 * (uint64_t)i + k];
    for (int k = 0; k < 32; k++) dom[k] = domain32[(uint64_t)i * domain_stride + k];
    attestation_signing_root(d, dom, o);
    for (int k = 0; k < 32; k++) out32[32 * (uint64_t)i + k] = o[k];
}
}  // namespace b2

// ------------------------------------------------------------------------------------------ SSZ wire decode of Attestation (SURVEY.md section 8(f)-3)
// Attestation (pos-evolution.md:714-717) on the wire: [u32 offset of aggregation_bits = 228][AttestationData, 128 B]
// [signature, 96 B][Bitlist[MAX_VALIDATORS_PER_COMMITTEE] bytes].  A Bitlist carries its length as a delimiter: the highest set
// bit of its last byte (:715); that byte may not be zero.  One warp per attestation: the lanes copy the fixed part, lane 0 finds
// the delimiter, the lanes write the bit row with the delimiter cleared and zero padding up to bits_stride bytes.
// status: 0 ok, 1 malformed container (too short / wrong offset), 2 empty bitlist or missing delimiter, 3 more than max_bits bits.
namespace b2 {
#define B2_ATT_FIXED 228u
// The container and delimiter checks of the encoding w = wire + begin, wire[begin .. end): the status above; nbits = the Bitlist's length
// in bits once the delimiter is found (statuses 0 and 3).  Shared by k_attestations_decode and the intake (intake.cuh).
__device__ __forceinline__ int32_t att_wire_parse(const uint8_t* w, uint32_t begin, uint32_t end, uint32_t bits_stride, uint32_t max_bits,
                                                  uint32_t& nbits) {
    if (end < begin || end - begin < B2_ATT_FIXED) return 1;
    const uint32_t o = (uint32_t)w[0] | ((uint32_t)w[1] << 8) | ((uint32_t)w[2] << 16) | ((uint32_t)w[3] << 24);
    const uint32_t nbytes = end - begin - B2_ATT_FIXED;
    if (o != B2_ATT_FIXED) return 1;
    if (nbytes == 0 || w[end - begin - 1] == 0) return 2;
    const uint32_t last = w[end - begin - 1];
    const uint32_t top = 31u - (uint32_t)__clz((int)last);          // position of the delimiter bit in the last byte
    nbits = 8 * (nbytes - 1) + top;
    return nbits > max_bits || (nbits + 7) / 8 > bits_stride ? 3 : 0;
}

__global__ void __launch_bounds__(128) k_attestations_decode(const uint8_t* __restrict__ wire, const uint32_t* __restrict__ woff, uint32_t n,
                                                              uint32_t bits_stride, uint32_t max_bits, uint8_t* bits_out, uint32_t* bit_len_out,
                                                              uint8_t* data128_out, uint8_t* sig96_out, int32_t* status_out) {
    const uint32_t a = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (a >= n) return;
    const uint32_t begin = woff[a], end = woff[a + 1];
    const uint8_t* w = wire + begin;
    uint8_t* brow = bits_out + (uint64_t)a * bits_stride;
    for (uint32_t k = lane; k < bits_stride; k += 32) brow[k] = 0;
    uint32_t nbits = 0;
    const int32_t st = att_wire_parse(w, begin, end, bits_stride, max_bits, nbits);
    if (st == 0) {
        for (uint32_t k = lane; k < 128; k += 32) data128_out[128 * (uint64_t)a + k] = w[4 + k];
        for (uint32_t k = lane; k < 96; k += 32) sig96_out[96 * (uint64_t)a + k] = w[132 + k];
        const uint32_t full = nbits >> 3;                                   // bytes that carry 8 payload bits
        __syncwarp();
        for (uint32_t k = lane; k < full; k += 32) brow[k] = w[B2_ATT_FIXED + k];
        if (lane == 0 && (nbits & 7u)) brow[full] = w[B2_ATT_FIXED + full] & (uint8_t)((1u << (nbits & 7u)) - 1u);
    } else {
        for (uint32_t k = lane; k < 128; k += 32) data128_out[128 * (uint64_t)a + k] = 0;
        for (uint32_t k = lane; k < 96; k += 32) sig96_out[96 * (uint64_t)a + k] = 0;
        nbits = 0;
    }
    if (lane == 0) {
        bit_len_out[a] = nbits;
        status_out[a] = st;
    }
}
}  // namespace b2

// ------------------------------------------------------------------------------------------ participation flags + proposer-reward numerators (SURVEY.md section 8(f)-2)
// The bookkeeping loop of process_attestation (pos-evolution.md:745-749): for every attesting index and every
// flag the attestation earns, set the flag if it is not set yet and credit get_base_reward(index) * weight to THIS
// attestation's proposer_reward_numerator.  Which attestation of a batch gets the credit matters (the numerator is divided
// per attestation, :752-754), so the parallel form is order-exact like K7: phase 1 elects, per (validator, flag), the
// earliest accepted attestation of the list that earns the still-unset flag (atomicMin on its list position); phase 2 sums
// the rewards of the elections each attestation won; phase 3 sets the flags and re-arms the election table.
namespace b2 {
__device__ __forceinline__ bool part_member(const uint32_t* members, const uint32_t* off, const uint8_t* bits, uint32_t stride, uint32_t a, uint32_t j,
                                            uint32_t& v) {
    if (!((bits[(uint64_t)a * stride + (j >> 3)] >> (j & 7)) & 1)) return false;
    v = members[off[a] + j];
    return true;
}
__global__ void __launch_bounds__(128) k_part_phase1(const uint32_t* __restrict__ members, const uint32_t* __restrict__ off,
                                                      const uint8_t* __restrict__ bits, uint32_t stride, const uint8_t* __restrict__ flag_mask,
                                                      const uint8_t* __restrict__ accept, uint32_t n_agg, const uint8_t* __restrict__ part,
                                                      uint32_t* first) {
    const uint32_t a = blockIdx.x;
    if (a >= n_agg || (accept && !accept[a])) return;
    const uint32_t mask = flag_mask[a] & 7u, size = off[a + 1] - off[a];
    uint32_t v;
    for (uint32_t j = threadIdx.x; j < size; j += blockDim.x)
        if (part_member(members, off, bits, stride, a, j, v)) {
            const uint32_t need = mask & ~(uint32_t)part[v];
#pragma unroll
            for (int f = 0; f < 3; f++)
                if ((need >> f) & 1u) atomicMin(&first[3 * (uint64_t)v + f], a);
        }
}
// weights = PARTICIPATION_FLAG_WEIGHTS (14, 26, 14); reward unit = (effective_balance / increment) * base_reward_per_increment
__global__ void __launch_bounds__(128) k_part_phase2(const uint32_t* __restrict__ members, const uint32_t* __restrict__ off,
                                                      const uint8_t* __restrict__ bits, uint32_t stride, const uint8_t* __restrict__ flag_mask,
                                                      const uint8_t* __restrict__ accept, uint32_t n_agg, const uint32_t* __restrict__ first,
                                                      const uint64_t* __restrict__ eff, unsigned long long increment, unsigned long long per_increment,
                                                      unsigned long long* numerator) {
    __shared__ unsigned long long red[4];
    const uint32_t a = blockIdx.x;
    if (a >= n_agg) return;
    unsigned long long sum = 0;
    if (!accept || accept[a]) {
        const uint32_t mask = flag_mask[a] & 7u, size = off[a + 1] - off[a];
        uint32_t v;
        for (uint32_t j = threadIdx.x; j < size; j += blockDim.x)
            if (part_member(members, off, bits, stride, a, j, v)) {
                const unsigned long long base = (eff[v] / increment) * per_increment;
                if ((mask & 1u) && first[3 * (uint64_t)v + 0] == a) sum += base * 14ull;
                if ((mask & 2u) && first[3 * (uint64_t)v + 1] == a) sum += base * 26ull;
                if ((mask & 4u) && first[3 * (uint64_t)v + 2] == a) sum += base * 14ull;
            }
    }
#pragma unroll
    for (int d = 16; d >= 1; d >>= 1) sum += __shfl_down_sync(B2_FULL_MASK, sum, d);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = sum;
    __syncthreads();
    if (threadIdx.x == 0) numerator[a] = red[0] + red[1] + red[2] + red[3];
}
__global__ void __launch_bounds__(128) k_part_phase3(const uint32_t* __restrict__ members, const uint32_t* __restrict__ off,
                                                      const uint8_t* __restrict__ bits, uint32_t stride, const uint8_t* __restrict__ flag_mask,
                                                      const uint8_t* __restrict__ accept, uint32_t n_agg, uint32_t* first, uint32_t* part_words) {
    const uint32_t a = blockIdx.x;
    if (a >= n_agg || (accept && !accept[a])) return;
    const uint32_t mask = flag_mask[a] & 7u, size = off[a + 1] - off[a];
    uint32_t v;
    for (uint32_t j = threadIdx.x; j < size; j += blockDim.x)
        if (part_member(members, off, bits, stride, a, j, v)) {
            uint32_t won = 0;
#pragma unroll
            for (int f = 0; f < 3; f++)
                if (((mask >> f) & 1u) && first[3 * (uint64_t)v + f] == a) {
                    won |= 1u << f;
                    first[3 * (uint64_t)v + f] = 0xffffffffu;       // single writer: only the elected attestation resets
                }
            if (won) atomicOr(&part_words[v >> 2], won << (8 * (v & 3)));
        }
}
}  // namespace b2

// ------------------------------------------------------------------------------------------ FFG balance sums (SURVEY.md section 8(f)-2)
// The three u64 sums process_justification_and_finalization feeds to weigh_justification_and_finalization
// (pos-evolution.md:793-803): total active balance, and the balance of the unslashed validators that carry
// `flag` in the current / previous epoch participation table (get_unslashed_participating_indices + get_total_balance).
// Registry flag byte: bit0 active in the current epoch, bit1 slashed, bit2 active in the previous epoch.  22 B per validator,
// one grid-stride pass, warp-shuffle + one atomicAdd per warp.  out[0] total active, out[1] current, out[2] previous,
// out[3] total active AND unslashed (the essay's prose reading of get_total_active_balance, :809).
namespace b2 {
__global__ void __launch_bounds__(256) k_ffg_balances(uint64_t n, const unsigned long long* __restrict__ eff, const uint8_t* __restrict__ flags,
                                                       const uint8_t* __restrict__ part_cur, const uint8_t* __restrict__ part_prev, uint32_t flag_bit,
                                                       unsigned long long* out) {
    unsigned long long s[4] = {0ull, 0ull, 0ull, 0ull};
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
        const uint32_t f = flags[i];
        const unsigned long long e = eff[i];
        const bool unslashed = !(f & 2u);
        if (f & 1u) {
            s[0] += e;
            if (unslashed) s[3] += e;
            if (unslashed && part_cur && ((part_cur[i] >> flag_bit) & 1u)) s[1] += e;
        }
        if ((f & 4u) && unslashed && part_prev && ((part_prev[i] >> flag_bit) & 1u)) s[2] += e;
    }
#pragma unroll
    for (int k = 0; k < 4; k++) {
#pragma unroll
        for (int d = 16; d; d >>= 1) s[k] += __shfl_down_sync(0xffffffffu, s[k], d);
        if ((threadIdx.x & 31) == 0 && s[k]) atomicAdd(&out[k], s[k]);
    }
}
}  // namespace b2

// ------------------------------------------------------------------------------------------ fork-choice variants (SURVEY.md section 8(f)-4)
// on_attester_slashing (pos-evolution.md:1447-1461): the validators in BOTH attesting-index lists become
// equivocating (Store.equivocating_indices, :897) and stop counting in get_weight (:1411-1413).  One thread per element of the
// first (sorted) list, binary search in the second.
namespace b2 {
__global__ void __launch_bounds__(128) k_mark_equivocating(const uint32_t* __restrict__ idx1, uint32_t n1, const uint32_t* __restrict__ idx2, uint32_t n2,
                                                            uint64_t n_val, uint8_t* equiv) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n1) return;
    const uint32_t v = idx1[i];
    uint32_t lo = 0, hi = n2;
    while (lo < hi) {
        uint32_t mid = (lo + hi) >> 1;
        if (idx2[mid] < v) lo = mid + 1; else hi = mid;
    }
    if (lo < n2 && idx2[lo] == v && v < n_val) equiv[v] = 1;
}
}  // namespace b2
