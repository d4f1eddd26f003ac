// b200pos.cu -- C ABI (include/b200pos.h) over the kernels in kernels.cuh.  Single translation
// unit -> libb200pos.so (nvcc -gencode arch=compute_90a,code=sm_90a).  No CPU fallback anywhere.
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <nvtx3/nvToolsExt.h>      // header-only NVTX v3: every C-ABI call is a named range in Nsight Systems / ncu --nvtx timelines

#include <algorithm>
#include <new>
#include <vector>

#include "../../include/b200pos.h"
#include "kernels.cuh"
#include "gather.cuh"
#include "rlc.cuh"
#include "aggverify.cuh"
#include "syncagg.cuh"
#include "slasher.cuh"
#include "pack.cuh"
#include "ssz.cuh"
#include "tree.cuh"
#include "votes.cuh"
#include "intake.cuh"
#include "single_intake.cuh"
#include "aggintake.cuh"
#include "blockatt.cuh"
#include "blockatt_electra.cuh"
#include "syncmsg.cuh"
#include "synccontrib.cuh"

using namespace b2;

// A device allocation with one owner: freed on destruction, moved (never copied) between owners, and passed to kernels and copies
// as whatever pointer type they take.  cudaFree waits for the device, so replacing a buffer that queued work still reads is safe.
struct dbuf {
    void* p = nullptr;
    size_t cap = 0;
    dbuf() = default;
    dbuf(dbuf&& o) noexcept : p(o.p), cap(o.cap) { o.p = nullptr, o.cap = 0; }
    dbuf& operator=(dbuf o) noexcept {      // the previous allocation leaves with `o`
        std::swap(p, o.p);
        std::swap(cap, o.cap);
        return *this;
    }
    ~dbuf() {
        if (p) cudaFree(p);
    }
    explicit operator bool() const { return p != nullptr; }
    template <class T> operator T*() const { return static_cast<T*>(p); }
};

// validator registry, latest messages and participation flags: n_val entries each, replaced together by b2_registry_load
struct registry_tables {
    dbuf records, valid, eff, flags;          // u32[24] affine pubkey record, u8 KeyValidate, u64 effective balance, u8 flags
    dbuf lmd_key, lmd_block, equiv;           // u64 epoch << 32 | 0xffffffff (0 = no message), u32 block, u8 equivocating
    dbuf part[2], part_first;                 // epoch participation flags (0 = current, 1 = previous), per-(validator, flag) election table
};
// The shared-memory budgets of fork choice: the tree phase (227 KB per block minus the tree kernels' static shared memory) and the vote
// scatter's per-CTA bins
constexpr int TREE_SMEM_BYTES = 226 * 1024;
constexpr int BINS_SMEM_BYTES = 200 * 1024;

// The kernels a tree runs, a function of its size alone (tree_form_of)
struct tree_form {
    bool smem_tree;         // the tree phase in shared memory (ghost_tree_smem), else the generic form on global memory
    bool work_list;         // ... with the work list of the marking phase
    size_t tree_smem;       // dynamic shared memory of the tree phase
    bool smem_bins;         // the vote scatter's bins in shared memory (k_ghost_votes_smem), else global atomics (k_ghost_votes)
};
// The shared-memory tree phase holds votes/prefix/weights u64[n+1], the packed word u32[n] and marks u32[n+1] in TREE_SMEM_BYTES, at most
// 15 elements per thread; when it still fits, the launch also reserves the work list u32[n].  The bins are u64[n].
static tree_form tree_form_of(uint32_t n) {
    const size_t base = ((size_t)n + 1) * 8 + (size_t)n * 8 + 8, with_list = base + (size_t)n * 4;
    const bool smem = base <= TREE_SMEM_BYTES && n <= 15 * 1024, list = smem && with_list <= TREE_SMEM_BYTES;
    return {smem, list, !smem ? 0 : list ? with_list : base, (size_t)n * 8 <= BINS_SMEM_BYTES};
}

// block tree (b2_tree_load): its form and the tables that form reads, in pre-order
struct tree_tables {
    tree_form form = {};
    dbuf pre, inv, head;                              // u32
    dbuf votes, weight;                               // u64
    dbuf packed;                                      // shared-memory form: u32 size | rank << 15 | keep << 31
    dbuf size_keep, rank, next;                       // generic form: u32 size | keep << 31, u32 root rank, u32[n+1] marks
    dbuf prefix, w2;                                  // generic form: u64[n+1] prefix sums, u64 weights
    // per block id, so that b2_tree_add / _prune / _set_viable change the tree on the device (tree.cuh); `pre` above is per id too
    dbuf size, rank_id, parent, root, viable;         // u32 subtree size, u32 rank of (root, id), u32 parent, u8[32] root, u8 viability
    dbuf slot;                                        // u64 block slot (read by the attestation intake)
    dbuf pre_b, size_b, rank_b, parent_b, root_b, viable_b, slot_b;      // the other side of the out-of-place steps (prune, grid insert)
    dbuf scan, scan2, map;                            // u32[n+1] prefix-count scratch, u32[n] prune map
};

// sync committees (b2_sync_committee_load): n committees of `size` keys, replaced together
struct sync_tables {
    dbuf records, valid;       // u32[24] affine record and u8 KeyValidate per position, committee after committee
    dbuf sum, sum_status;      // per committee: Jacobian sum of its valid keys (u32[36]), k_g1_segment_sum's status byte
    uint32_t size = 0, n = 0;
};

// slasher (b2_slasher_init): span tables and first-vote ids per (validator, epoch of the ring), per-column counts and root log
// (slasher.cuh), and the ids of the aggregates of the update in flight
struct slasher_tables {
    dbuf min_span, max_span, first_id, count, root, agg_id;
    uint64_t n_val = 0, n_rows = 0;      // validators of the registry; rows held, for validators v_begin .. v_begin + n_rows - 1
    uint32_t v_begin = 0;
    uint32_t H = 0, K = 0, cur = 0;      // H == 0: not initialised
};

// hash_tree_root (ssz.cuh): the validators tree's node cache over C leaves (heap layout, 2C nodes of 8 words) and the scratch tree of
// b2_ssz_chunks_root
struct ssz_tables {
    dbuf cache;
    uint64_t n = 0, C = 0;      // C == 0: no cache
    dbuf chunks;
};

struct vslot {
    dbuf haff, hflag, pkjac, pkst, saff, sflag, f, sumjac;
    dbuf g2aff, g2st;                                      // the slot's own decompressed signatures (pipelined epochs)
    uint64_t n_sig_tail = 0;                               // signatures of the epoch whose segment sums the tail still has to run
    bool segsum_pending = false;
    dbuf pkjac_r, rscal, sg_aff, sg_flag, f_g, gpass;      // RLC batch mode: [r]PK, r, per-group signature sums, group Miller values / verdicts
    cudaEvent_t ev_join0 = nullptr, ev_join1 = nullptr, ev_seg = nullptr, ev_tail_done = nullptr, ev_fork = nullptr, ev_in = nullptr;
    cudaStream_t s_tail = nullptr;      // the slot's own tail stream: tails of consecutive epochs overlap each other
    // the slot's own side streams (hash-to-G2; pubkey aggregation + first Miller loop).  With ONE pair shared by all slots the
    // latency-bound side chains of consecutive epochs serialise (6 + 10 ms per epoch) -- invisible behind a 32 ms decompression,
    // but the bound of the step once an epoch is sharded over 8 GPUs and its decompression takes 3.7 ms.
    cudaStream_t s_aux[2] = {nullptr, nullptr};
};

struct b2_ctx {
    int device = 0;
    int n_sm = 132;
    cudaStream_t s_main = nullptr;
    // pipelined epochs: the decompression kernels of consecutive epochs alternate between two streams, so the blocks of epoch k+1 fill
    // the SMs that epoch k's last, partial wave leaves idle (a rank's share of a sharded epoch is 1.7 waves at N = 8: 5.04 ms instead of
    // 3.65 ms per 131 072 signatures when the kernels run back to back on one stream)
    cudaStream_t s_dec[4] = {nullptr, nullptr, nullptr, nullptr};
    unsigned n_dec_streams = 2;                       // B2_DEC_STREAMS (2..4)
    // Measured on an earlier GPU, not re-measured on the H100: one rank's share at N = 8 / 4: 5.45 vs 5.97 and 9.75 vs 10.07 ms per epoch; at N = 1 (13.8 waves) the
    // overlap costs 0.3 ms instead, so the alternation is used only for decompressions of fewer than 6 waves (B2_DEC_ALTERNATE=0/1 forces)
    int dec_alternate = -1;                           // -1 auto, 0 never, 1 always
    unsigned dec_turn = 0;
    cudaEvent_t ev_votes_done = nullptr, ev_lmd_done = nullptr;
    cudaEvent_t ev_equiv_done = nullptr;             // the last equivocation mark enqueued (b2_slasher_discount_dev, b2_equivocating_merge_dev)
    cudaEvent_t ev_intake = nullptr;                 // the last attestation intake enqueued: the next one re-uses its scratch
    vslot slot[B2_EPOCH_SLOTS];
    char err[512] = {0};
    uint64_t launches = 0;
    uint64_t n_val = 0;
    registry_tables reg;
    // fork-choice variants: votes older than fc_min_key (epoch << 32) expire; v1.3 get_weight skips slashed validators
    // threads per block of the thread-per-aggregate kernels when they run under the epoch pipeline (see launch_miller)
    unsigned tail_block = 128;
    bool epoch_team = false;   // b2_epoch_set_pairing_form
    unsigned k2_block = 32;    // threads per aggregate of k_g1_aggregate under the epoch pipeline (B2_K2_BLOCK: 32/64/128)
    // K2 through the TMA-staged gather kernel (gather.cuh) instead of the LDG form; B2_K2_TMA=0 selects the LDG form (A/B)
    bool k2_tma = true;
    // FastAggregateVerify mode: 0 = one pairing check per aggregate; 1 = random-linear-combination batches of B2_RLC_GROUP
    // aggregates with per-aggregate fallback (b2_set_verify_mode); d_rlc_seed = the verifier's secret 32-byte seed
    int verify_mode = 0;
    dbuf d_rlc_seed;
    int pairing_form = 0;      // 0: team kernels for the synchronous calls, thread-per-aggregate under the pipeline; 1: always team; 2: always thread
    // threads per block of k_g2_decompress: its blocks fill the register file, so a smaller block is what a pairing warp of the
    // previous epoch displaces when the two overlap
    unsigned dec_block = 128;
    // one-launch get_head (k_get_head_fused): ticket counter, and the result slot in mapped pinned host memory (head, sequence)
    bool head_fused = true;                           // B2_HEAD_FUSED=0: the two-launch + memcpy form of round 1
    dbuf d_ticket;
    volatile uint32_t* h_head = nullptr;
    uint32_t* d_head_host = nullptr;
    uint32_t head_seq = 0;
    // multi-GPU get_head over NVLink peer memory (b2_fc_exchange_*): this rank's exchange block = accumulators 2 x n_blocks u64 followed by
    // flag rows 2 x B2_MAX_PEERS u32; peers' blocks opened through CUDA IPC
    dbuf fc_block;
    uint32_t fc_blocks_cap = 0;                       // n_blocks the block was sized for
    void* fc_peer[B2_MAX_PEERS] = {nullptr};
    int fc_rank = -1, fc_world = 0;
    uint32_t fc_seq = 0;
    dbuf d_dbg;                                       // clock64() stamps of the last get_head's phases (b2_debug_head_clocks)
    dbuf d_guard;                                     // device-side input guard word (kernels.cuh GuardBits), read by b2_guard_flags
    unsigned long long fc_min_key = 0;
    int fc_exclude_slashed = 0;
    // block tree
    uint32_t n_blocks = 0;
    tree_tables tree;
    // scratch
    dbuf sc_pkjac, sc_pkst, sc_haff, sc_hflag, sc_g2aff, sc_g2st, sc_rec, sc_val, sc_shuf, sc_pivot;
    // bls.AggregateVerify: signature points / flags, partial products and status words of the (block, set) runs, offsets-malformed
    // word; and its own side streams and events, so that it never re-records an event an epoch in flight waits on
    dbuf sc_av_saff, sc_av_sflag, sc_av_f, sc_av_st, sc_av_bad;
    cudaStream_t s_av[2] = {nullptr, nullptr};
    cudaEvent_t ev_av[3] = {nullptr, nullptr, nullptr};
    std::vector<dbuf> stage;                          // the synchronous entry points' host inputs and outputs (struct staging)
    sync_tables sync;
    slasher_tables sl;
    ssz_tables ssz;
    // per-call scratch (struct scratch) of the attestation and aggregated-attestation intakes, block attestations, sync committee
    // messages, sync committee contributions and block packing
    std::vector<dbuf> in, api, ba, scm, scc, pk;
};

struct nvtx_scope {
    explicit nvtx_scope(const char* name) { nvtxRangePushA(name); }
    ~nvtx_scope() { nvtxRangePop(); }
};
#define B2_NVTX nvtx_scope nvtx_scope_(__func__)

static int fail_cuda(b2_ctx* c, cudaError_t e, const char* what) {
    cudaGetLastError();      // consume a pending non-sticky error (a failed cudaMalloc sets one), so the next CKL sees only its own launch
    if (c) snprintf(c->err, sizeof(c->err), "%s: %s", what, cudaGetErrorString(e));
    return B2_ECUDA;
}
#define CK(call)                                                   \
    do {                                                           \
        cudaError_t e_ = (call);                                   \
        if (e_ != cudaSuccess) return fail_cuda(ctx, e_, #call);   \
    } while (0)
#define CKL(ctx_)                                                          \
    do {                                                                   \
        cudaError_t e_ = cudaGetLastError();                               \
        if (e_ != cudaSuccess) return fail_cuda(ctx_, e_, "kernel launch"); \
        (ctx_)->launches++;                                                \
    } while (0)
#define REQUIRE(cond, msg)                                         \
    do {                                                           \
        if (!(cond)) {                                             \
            if (ctx) snprintf(ctx->err, sizeof(ctx->err), "%s", msg); \
            return B2_EINVAL;                                      \
        }                                                          \
    } while (0)

static int ensure(b2_ctx* ctx, dbuf& b, size_t bytes) {
    if (bytes <= b.cap && b.p) return B2_OK;
    if (b.p) CK(cudaFree(b.p));
    b.p = nullptr;
    b.cap = 0;
    size_t want = std::max<size_t>(bytes, 256);
    CK(cudaMalloc(&b.p, want));
    b.cap = want;
    return B2_OK;
}

// One call's device buffers from a grow-only list: the i-th request gets bufs[i], grown as ensure grows it, so a call that makes its
// requests in a fixed order finds each buffer where it left it.  The first error is kept in rc and makes every later request a no-op
// (a null pointer), so a caller checks rc once after its requests and before its first memset or launch.
struct scratch {
    b2_ctx* ctx;
    std::vector<dbuf>& bufs;
    size_t used = 0;
    int rc = B2_OK;
    scratch(b2_ctx* c, std::vector<dbuf>& b) : ctx(c), bufs(b) {}
    void* buf(size_t bytes) {
        if (rc) return nullptr;
        if (used == bufs.size()) bufs.emplace_back();
        dbuf& b = bufs[used++];
        rc = ensure(ctx, b, bytes);
        return rc ? nullptr : b.p;
    }
    // p = a buffer of `count` T and `pad` bytes past them
    template <class T> void operator()(T*& p, size_t count, size_t pad = 0) { p = static_cast<T*>(buf(count * sizeof(T) + pad)); }
};

// One synchronous call's host traffic on s_main.  in() uploads a host array into the call's next staging buffer (ctx->stage);
// out() registers a host output with the device buffer that holds it (by default a staging buffer of its own); finish() copies every
// output to host memory, synchronises, and only if all of that succeeded writes the caller's buffers.  As in scratch, the first error
// makes every later step a no-op, so a caller checks rc once before its launches and returns finish().
struct staging : scratch {
    struct output {
        void* host;
        const void* dev;
        size_t bytes;
    };
    std::vector<output> outs;
    explicit staging(b2_ctx* c) : scratch(c, c->stage) {}
    // `pad` bytes past the end are allocated but not copied
    template <class T> const T* in(const T* host, size_t count, size_t pad = 0) {
        void* d = buf(count * sizeof(T) + pad);
        cudaError_t e = d && count ? cudaMemcpyAsync(d, host, count * sizeof(T), cudaMemcpyHostToDevice, ctx->s_main) : cudaSuccess;
        if (e != cudaSuccess) rc = fail_cuda(ctx, e, "staging upload");
        return static_cast<const T*>(d);
    }
    template <class T> T* out(T* host, size_t count) {
        T* d = static_cast<T*>(buf(count * sizeof(T)));
        out(host, d, count);
        return d;
    }
    template <class T> void out(T* host, const void* dev, size_t count) {
        if (!rc) outs.push_back({host, dev, count * sizeof(T)});
    }
    int finish() {
        if (rc) return rc;
        size_t total = 0;
        for (const output& o : outs) total += o.bytes;
        std::vector<uint8_t> tmp(total);
        uint8_t* h = tmp.data();
        for (const output& o : outs) {
            CK(cudaMemcpyAsync(h, o.dev, o.bytes, cudaMemcpyDeviceToHost, ctx->s_main));
            h += o.bytes;
        }
        CK(cudaStreamSynchronize(ctx->s_main));
        h = tmp.data();
        for (const output& o : outs) {
            memcpy(o.host, h, o.bytes);
            h += o.bytes;
        }
        return B2_OK;
    }
};

// Argument checks.  An entry point with a host and a device form has one check_X, called by both, for every condition on the arguments
// both receive and on the tables it needs; the host form adds only the checks that read its host arrays (check_offsets .. check_batch).
// `what` names the entry point in the message, which is the same whichever form was called.
static int reject(b2_ctx* ctx, const char* what, const char* why) {
    snprintf(ctx->err, sizeof(ctx->err), "%s: %s", what, why);
    return B2_EINVAL;
}
// the offsets off[0..n] start at 0 and never decrease
static int check_offsets(b2_ctx* ctx, const uint32_t* off, uint32_t n, const char* what, const char* name = "off") {
    if (off[0] == 0 && std::is_sorted(off, off + n + 1)) return B2_OK;
    snprintf(ctx->err, sizeof(ctx->err), "%s: %s must start at 0 and never decrease", what, name);
    return B2_EINVAL;
}
// a wire batch's item offsets woff[0..n]: check_offsets, and the last item ends within the wire
static int check_wire(b2_ctx* ctx, const uint32_t* woff, uint32_t n, uint64_t wire_len, const char* what) {
    if (int rc = check_offsets(ctx, woff, n, what, "woff")) return rc;
    return woff[n] <= wire_len ? B2_OK : reject(ctx, what, "woff ends past the wire");
}
// the member offsets off[0..n] of n committees: check_offsets, and no committee is wider than its 8 * bits_stride bit row
static int check_committees(b2_ctx* ctx, const uint32_t* off, uint32_t n, uint32_t bits_stride, const char* what) {
    if (int rc = check_offsets(ctx, off, n, what)) return rc;
    for (uint32_t c = 0; c < n; c++)
        if (off[c + 1] - off[c] > 8ull * bits_stride) return reject(ctx, what, "a committee is larger than 8 * bits_stride");
    return B2_OK;
}
// a committee batch: check_committees, and every member addresses one of `limit` validators
static int check_batch(b2_ctx* ctx, const uint32_t* members, const uint32_t* off, uint32_t bits_stride, uint32_t n_agg, uint64_t limit, const char* what) {
    if (int rc = check_committees(ctx, off, n_agg, bits_stride, what)) return rc;
    for (uint32_t i = 0; i < off[n_agg]; i++)
        if (members[i] >= limit) return reject(ctx, what, "member index outside the registry");
    return B2_OK;
}
#define B2_TEAM_SMEM (B2_TEAMS_PER_WARP * sizeof(team_ws))
static inline unsigned blocks_for(uint64_t n, unsigned t) { return (unsigned)((n + t - 1) / t); }
// true when environment variable `name` is set; *v = its value as atoi reads it
static bool env_int(const char* name, int* v) {
    const char* s = getenv(name);
    if (s) *v = atoi(s);
    return s != nullptr;
}
static bool is_block_knob(int v) { return v == 32 || v == 64 || v == 128; }

extern "C" {

int b2_init(int device, b2_ctx** out) {
    B2_NVTX;
    if (!out) return B2_EINVAL;
    *out = nullptr;
    // 8 pipeline slots x (tail + 2 side streams) + main/copy/fork-choice streams: more streams than the default 8 hardware queues,
    // whose aliasing creates false dependencies between slots.  Only effective when this is the first CUDA call of the process
    // (bench.py and the package __init__ also set it before torch initialises CUDA).
    setenv("CUDA_DEVICE_MAX_CONNECTIONS", "32", 0);
    int count = 0;
    if (cudaGetDeviceCount(&count) != cudaSuccess || count <= 0 || device < 0 || device >= count) return B2_ENODEVICE;
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, device) != cudaSuccess) return B2_ENODEVICE;
    if (prop.major != 9 || prop.minor != 0) return B2_ENODEVICE;      // sm_90a cubin only: loads on compute capability 9.0
    if (cudaSetDevice(device) != cudaSuccess) return B2_ENODEVICE;
    b2_ctx* ctx = new (std::nothrow) b2_ctx();
    if (!ctx) return B2_ENOMEM;
    ctx->device = device;
    // side streams get the highest priority: their kernels are small and latency-bound and must be scheduled as soon
    // as SM resources free up while a grid-filling kernel (signature decompression) occupies the main stream
    int prio_lo = 0, prio_hi = 0;
    cudaDeviceGetStreamPriorityRange(&prio_lo, &prio_hi);
    cudaError_t e = cudaStreamCreateWithPriority(&ctx->s_main, cudaStreamNonBlocking, prio_lo);
    for (int i = 0; i < 4 && e == cudaSuccess; i++) e = cudaStreamCreateWithPriority(&ctx->s_dec[i], cudaStreamNonBlocking, prio_lo);
    for (int i = 0; i < B2_EPOCH_SLOTS && e == cudaSuccess; i++) {
        e = cudaStreamCreateWithPriority(&ctx->slot[i].s_tail, cudaStreamNonBlocking, prio_hi);
        for (int k = 0; k < 2 && e == cudaSuccess; k++) e = cudaStreamCreateWithPriority(&ctx->slot[i].s_aux[k], cudaStreamNonBlocking, prio_hi);
    }
    for (int k = 0; k < 2 && e == cudaSuccess; k++) e = cudaStreamCreateWithPriority(&ctx->s_av[k], cudaStreamNonBlocking, prio_hi);
    for (int k = 0; k < 3 && e == cudaSuccess; k++) e = cudaEventCreateWithFlags(&ctx->ev_av[k], cudaEventDisableTiming);
    if (e == cudaSuccess) e = cudaEventCreateWithFlags(&ctx->ev_lmd_done, cudaEventDisableTiming);
    if (e == cudaSuccess) e = cudaEventCreateWithFlags(&ctx->ev_votes_done, cudaEventDisableTiming);
    if (e == cudaSuccess) e = cudaEventCreateWithFlags(&ctx->ev_equiv_done, cudaEventDisableTiming);
    if (e == cudaSuccess) e = cudaEventCreateWithFlags(&ctx->ev_intake, cudaEventDisableTiming);
    for (int i = 0; i < B2_EPOCH_SLOTS && e == cudaSuccess; i++) {
        cudaEvent_t* evs[6] = {&ctx->slot[i].ev_join0, &ctx->slot[i].ev_join1, &ctx->slot[i].ev_seg, &ctx->slot[i].ev_tail_done, &ctx->slot[i].ev_fork,
                               &ctx->slot[i].ev_in};
        for (int k = 0; k < 6 && e == cudaSuccess; k++) e = cudaEventCreateWithFlags(evs[k], cudaEventDisableTiming);
    }
    if (e == cudaSuccess) e = cudaFuncSetAttribute(k_ghost_tree, cudaFuncAttributeMaxDynamicSharedMemorySize, TREE_SMEM_BYTES);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(k_ghost_votes_smem, cudaFuncAttributeMaxDynamicSharedMemorySize, BINS_SMEM_BYTES);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(k_g1_gather_tma<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 4 * (int)sizeof(gather_ws));
    if (e == cudaSuccess) e = cudaFuncSetAttribute(k_g1_gather_tma<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 4 * (int)sizeof(gather_ws));
    ctx->n_sm = prop.multiProcessorCount;
    if (e == cudaSuccess) e = cudaMalloc(&ctx->d_dbg.p, 32 * 8);
    if (e == cudaSuccess) e = cudaMemset(ctx->d_dbg, 0, 32 * 8);
    if (e == cudaSuccess) e = cudaMalloc(&ctx->d_ticket.p, 64);
    if (e == cudaSuccess) e = cudaMemset(ctx->d_ticket, 0, 64);
    if (e == cudaSuccess) e = cudaHostAlloc((void**)&ctx->h_head, 64, cudaHostAllocMapped);
    if (e == cudaSuccess) {
        memset((void*)ctx->h_head, 0, 64);
        e = cudaHostGetDevicePointer((void**)&ctx->d_head_host, (void*)ctx->h_head, 0);
    }
    if (e == cudaSuccess) e = cudaFuncSetAttribute(k_get_head_fused, cudaFuncAttributeMaxDynamicSharedMemorySize, TREE_SMEM_BYTES);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(k_get_head_fused_nvl, cudaFuncAttributeMaxDynamicSharedMemorySize, TREE_SMEM_BYTES);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(k_pack_committee, cudaFuncAttributeMaxDynamicSharedMemorySize, PACK_SMEM_ROWS);
    if (e == cudaSuccess) e = cudaMalloc(&ctx->d_rlc_seed.p, 32);
    if (e == cudaSuccess) e = cudaMemset(ctx->d_rlc_seed, 0, 32);
    if (e == cudaSuccess) e = cudaMalloc(&ctx->d_guard.p, 256);
    if (e == cudaSuccess) e = cudaMemset(ctx->d_guard, 0, 256);
    // diagnostic knobs (INTEGRATION.md); unset or out-of-range values keep the defaults, which are the measured best
    int v = 0;
    if (env_int("B2_DEC_STREAMS", &v) && v >= 2 && v <= 4) ctx->n_dec_streams = (unsigned)v;
    if (env_int("B2_DEC_ALTERNATE", &v)) ctx->dec_alternate = v != 0 ? 1 : 0;
    if (env_int("B2_TAIL_BLOCK", &v) && is_block_knob(v)) ctx->tail_block = (unsigned)v;
    if (env_int("B2_K2_BLOCK", &v) && is_block_knob(v)) ctx->k2_block = (unsigned)v;
    if (env_int("B2_DEC_BLOCK", &v) && is_block_knob(v)) ctx->dec_block = (unsigned)v;
    if (env_int("B2_K2_TMA", &v)) ctx->k2_tma = v != 0;
    if (env_int("B2_HEAD_FUSED", &v)) ctx->head_fused = v != 0;
    if (const char* form = getenv("B2_PAIRING_FORM")) ctx->pairing_form = !strcmp(form, "team") ? 1 : (!strcmp(form, "thread") ? 2 : 0);
    if (e != cudaSuccess) {
        b2_destroy(ctx);
        return B2_ECUDA;
    }
    *out = ctx;
    return B2_OK;
}

// also the failure path of b2_init: every handle may still be null
void b2_destroy(b2_ctx* ctx) {
    if (!ctx) return;
    cudaSetDevice(ctx->device);
    cudaDeviceSynchronize();
    for (int r = 0; r < B2_MAX_PEERS; r++)      // before this rank's own exchange block is freed
        if (ctx->fc_peer[r] && r != ctx->fc_rank) cudaIpcCloseMemHandle(ctx->fc_peer[r]);
    for (int i = 0; i < B2_EPOCH_SLOTS; i++) {
        vslot& V = ctx->slot[i];
        cudaEvent_t evs[6] = {V.ev_join0, V.ev_join1, V.ev_seg, V.ev_tail_done, V.ev_fork, V.ev_in};
        for (cudaEvent_t ev : evs)
            if (ev) cudaEventDestroy(ev);
        if (V.s_tail) cudaStreamDestroy(V.s_tail);
        for (int k = 0; k < 2; k++)
            if (V.s_aux[k]) cudaStreamDestroy(V.s_aux[k]);
    }
    if (ctx->s_main) cudaStreamDestroy(ctx->s_main);
    for (int i = 0; i < 4; i++)
        if (ctx->s_dec[i]) cudaStreamDestroy(ctx->s_dec[i]);
    for (int k = 0; k < 2; k++)
        if (ctx->s_av[k]) cudaStreamDestroy(ctx->s_av[k]);
    for (int k = 0; k < 3; k++)
        if (ctx->ev_av[k]) cudaEventDestroy(ctx->ev_av[k]);
    if (ctx->ev_lmd_done) cudaEventDestroy(ctx->ev_lmd_done);
    if (ctx->ev_votes_done) cudaEventDestroy(ctx->ev_votes_done);
    if (ctx->ev_equiv_done) cudaEventDestroy(ctx->ev_equiv_done);
    if (ctx->ev_intake) cudaEventDestroy(ctx->ev_intake);
    if (ctx->h_head) cudaFreeHost((void*)ctx->h_head);
    delete ctx;      // frees every device buffer
}

const char* b2_last_error(b2_ctx* ctx) { return ctx ? ctx->err : "null context"; }
uint64_t b2_launch_count(b2_ctx* ctx) { return ctx ? ctx->launches : 0; }
uint32_t b2_tree_size(b2_ctx* ctx) { return ctx ? ctx->n_blocks : 0; }
int b2_sync(b2_ctx* ctx) {
    B2_NVTX;
    REQUIRE(ctx, "null context");
    CK(cudaSetDevice(ctx->device));
    CK(cudaDeviceSynchronize());
    return B2_OK;
}

int b2_guard_flags(b2_ctx* ctx, uint32_t* flags_out) {
    B2_NVTX;
    REQUIRE(ctx && flags_out, "guard_flags: bad arguments");
    CK(cudaSetDevice(ctx->device));
    CK(cudaDeviceSynchronize());
    uint32_t f = 0;
    CK(cudaMemcpy(&f, ctx->d_guard, 4, cudaMemcpyDeviceToHost));
    CK(cudaMemset(ctx->d_guard, 0, 4));
    *flags_out = f;
    return B2_OK;
}

// ------------------------------------------------------------------------------------------ registry
int b2_registry_load(b2_ctx* ctx, const uint8_t* pk48, const uint64_t* eff, const uint8_t* flags, uint64_t n, uint8_t* pk_valid_out) {
    B2_NVTX;
    REQUIRE(ctx && pk48 && eff && flags && n > 0 && n < (1ull << 32), "registry_load: bad arguments");
    CK(cudaSetDevice(ctx->device));
    // The new tables are built aside and replace the old ones only once complete, so a failed load leaves the registry as it was.
    // Every allocation, the largest first, comes before the first read of the caller's arrays.
    registry_tables t;
    int rc;
    if ((rc = ensure(ctx, t.records, n * 96)) || (rc = ensure(ctx, t.valid, n)) || (rc = ensure(ctx, t.eff, n * 8)) || (rc = ensure(ctx, t.flags, n)) ||
        (rc = ensure(ctx, t.lmd_key, n * 8)) || (rc = ensure(ctx, t.lmd_block, n * 4)) ||
        (rc = ensure(ctx, t.equiv, (n + 3) & ~3ull)))      // whole words: k_slasher_discount marks by a 32-bit atomicOr
        return rc;
    staging st(ctx);
    const uint8_t* d_pk = st.in(pk48, n * 48);
    if (st.rc) return st.rc;
    cudaStream_t s = ctx->s_main;
    CK(cudaMemcpyAsync(t.eff, eff, n * 8, cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync(t.flags, flags, n, cudaMemcpyHostToDevice, s));
    CK(cudaMemsetAsync(t.lmd_key, 0, n * 8, s));
    CK(cudaMemsetAsync(t.lmd_block, 0, n * 4, s));
    CK(cudaMemsetAsync(t.equiv, 0, n, s));
    k_registry_load<<<blocks_for(n, 128), 128, 0, s>>>(d_pk, n, t.records, t.valid);
    CKL(ctx);
    if (pk_valid_out) st.out(pk_valid_out, t.valid, n);
    if ((rc = st.finish())) return rc;
    ctx->reg = std::move(t);        // the participation tables are dropped: t has none
    ctx->n_val = n;
    return B2_OK;
}

// bls.KeyValidate for n explicit pubkeys, without touching the registry (scratch buffers only)
int b2_key_validate(b2_ctx* ctx, const uint8_t* pk48, uint64_t n, uint8_t* valid_out) {
    B2_NVTX;
    REQUIRE(ctx && pk48 && valid_out && n > 0 && n < (1ull << 32), "key_validate: bad arguments");
    CK(cudaSetDevice(ctx->device));
    staging st(ctx);
    const uint8_t* d_pk = st.in(pk48, n * 48);
    int rc;
    if ((rc = st.rc) || (rc = ensure(ctx, ctx->sc_rec, n * 96 + 16)) || (rc = ensure(ctx, ctx->sc_val, n + 16))) return rc;
    k_g1_decompress_validate<<<blocks_for(n, 128), 128, 0, ctx->s_main>>>(d_pk, n, (uint32_t*)ctx->sc_rec.p, (uint8_t*)ctx->sc_val.p);
    CKL(ctx);
    st.out(valid_out, ctx->sc_val, n);
    return st.finish();
}

int b2_registry_update_balances(b2_ctx* ctx, const uint64_t* eff, const uint8_t* flags, uint64_t n) {
    B2_NVTX;
    REQUIRE(ctx && eff && flags && n == ctx->n_val && n > 0, "registry_update_balances: registry not loaded or size mismatch");
    CK(cudaSetDevice(ctx->device));
    CK(cudaMemcpyAsync(ctx->reg.eff, eff, n * 8, cudaMemcpyHostToDevice, ctx->s_main));
    CK(cudaMemcpyAsync(ctx->reg.flags, flags, n, cudaMemcpyHostToDevice, ctx->s_main));
    CK(cudaStreamSynchronize(ctx->s_main));
    return B2_OK;
}

// K2 launch: one warp per aggregate through the TMA-staged gather (wpb warps = aggregates per block), or the LDG form with
// `ldg_block` threads per aggregate
static int launch_k2(b2_ctx* ctx, const uint32_t* d_members, const uint32_t* d_off, const uint8_t* d_bits, uint32_t bits_stride, uint32_t n_agg,
                     uint32_t* d_pkjac, uint8_t* d_pkst, unsigned wpb, unsigned ldg_block, cudaStream_t s) {
    if (ctx->k2_tma) {
        k_g1_gather_tma<false><<<blocks_for(n_agg, wpb), wpb * 32, wpb * sizeof(gather_ws), s>>>(ctx->reg.records, d_members, d_off, d_bits, bits_stride, n_agg,
                                                                                             d_pkjac, d_pkst, ctx->n_val, ctx->d_guard, nullptr);
    } else {
        k_g1_aggregate<<<n_agg, ldg_block, 0, s>>>(ctx->reg.records, ctx->reg.valid, d_members, d_off, d_bits, bits_stride, n_agg, d_pkjac, d_pkst, ctx->n_val,
                                                   ctx->d_guard);
    }
    CKL(ctx);
    return B2_OK;
}

static int g1_aggregate_dev(b2_ctx* ctx, const uint32_t* d_members, const uint32_t* d_off, const uint8_t* d_bits, uint32_t bits_stride,
                            uint32_t n_agg, cudaStream_t s) {
    int rc;
    if ((rc = ensure(ctx, ctx->sc_pkjac, (size_t)n_agg * 144)) || (rc = ensure(ctx, ctx->sc_pkst, n_agg))) return rc;
    return launch_k2(ctx, d_members, d_off, d_bits, bits_stride, n_agg, (uint32_t*)ctx->sc_pkjac.p, (uint8_t*)ctx->sc_pkst.p, 4, 128, s);
}

int b2_g1_aggregate(b2_ctx* ctx, const uint32_t* members, const uint32_t* off, const uint8_t* bits, uint32_t bits_stride, uint32_t n_agg,
                    uint8_t* out48, uint8_t* status) {
    B2_NVTX;
    REQUIRE(ctx && members && off && bits && out48 && status && n_agg > 0 && bits_stride > 0, "g1_aggregate: bad arguments");
    REQUIRE(ctx->n_val > 0, "g1_aggregate: registry not loaded");
    int rc;
    if ((rc = check_batch(ctx, members, off, bits_stride, n_agg, ctx->n_val, "g1_aggregate"))) return rc;
    CK(cudaSetDevice(ctx->device));
    cudaStream_t s = ctx->s_main;
    staging st(ctx);
    const uint32_t* dm = st.in(members, off[n_agg], 4);
    const uint32_t* dof = st.in(off, (size_t)n_agg + 1);
    const uint8_t* db = st.in(bits, (size_t)n_agg * bits_stride, 16);
    uint8_t* d48 = st.out(out48, (size_t)n_agg * 48);
    if ((rc = st.rc) || (rc = g1_aggregate_dev(ctx, dm, dof, db, bits_stride, n_agg, s))) return rc;
    k_g1_compress<<<blocks_for(n_agg, 64), 64, 0, s>>>((const uint32_t*)ctx->sc_pkjac.p, n_agg, d48);
    CKL(ctx);
    st.out(status, ctx->sc_pkst, n_agg);
    return st.finish();
}

// The gather stage of K2 ALONE (no additions): XOR checksum of the records each aggregate selects.  form 1: TMA-staged
// (k_g1_gather_tma<true>), form 0: plain 128-bit loads (k_g1_gather_ldg_probe).  bench.py times it for `roofline.gather`.
int b2_gather_probe_dev(b2_ctx* ctx, const uint32_t* d_members, const uint32_t* d_off, const uint8_t* d_bits, uint32_t bits_stride, uint32_t n_agg,
                        int form, uint32_t* d_checksum_out, void* stream) {
    B2_NVTX;
    REQUIRE(ctx && d_members && d_off && d_bits && d_checksum_out && n_agg > 0 && bits_stride > 0 && (form == 0 || form == 1), "gather_probe_dev: bad arguments");
    REQUIRE(ctx->n_val > 0, "gather_probe: registry not loaded");
    CK(cudaSetDevice(ctx->device));
    cudaStream_t s = (cudaStream_t)stream;
    if (form == 1) {
        k_g1_gather_tma<true><<<blocks_for(n_agg, 4), 128, 4 * sizeof(gather_ws), s>>>(ctx->reg.records, d_members, d_off, d_bits, bits_stride, n_agg, nullptr,
                                                                                    nullptr, ctx->n_val, ctx->d_guard, d_checksum_out);
    } else {
        k_g1_gather_ldg_probe<<<n_agg, 128, 0, s>>>(ctx->reg.records, d_members, d_off, d_bits, bits_stride, n_agg, ctx->n_val, d_checksum_out);
    }
    CKL(ctx);
    return B2_OK;
}

// ------------------------------------------------------------------------------------------ bls.Aggregate
// front: stage 1 + 2 (decompress every signature, per-segment Jacobian sums into V.sumjac);  finish: stage 3 (one
// inversion per segment -> compressed bytes; with `handoff` also the affine point + subgroup-checked flag for verify_main).
// `seg_stream`: the stream the per-segment sums run on.  Same as `s` for the synchronous entry points.  Under the epoch pipeline it
// is the slot's TAIL stream: the decompressed points then live in the slot's own buffer and the caller's stream goes straight on to
// the next epoch's decompression instead of waiting ~2 ms for a 2 048-warp kernel that cannot fill the chip.
static int aggregate_front(b2_ctx* ctx, vslot& V, const uint8_t* d_sig96, const uint32_t* d_seg_off, uint32_t n_seg, uint64_t n_sig,
                           int32_t* d_seg_status, cudaStream_t s, bool own_buffers = false) {
    int rc;
    dbuf& aff = own_buffers ? V.g2aff : ctx->sc_g2aff;
    dbuf& st = own_buffers ? V.g2st : ctx->sc_g2st;
    if ((rc = ensure(ctx, aff, (size_t)n_sig * 192 + 16)) || (rc = ensure(ctx, st, n_sig + 16)) || (rc = ensure(ctx, V.sumjac, (size_t)n_seg * 288))) return rc;
    if (n_sig) {
        k_g2_decompress<<<blocks_for(n_sig, ctx->dec_block), ctx->dec_block, 0, s>>>(d_sig96, n_sig, (uint32_t*)aff.p, (uint8_t*)st.p);
        CKL(ctx);
    }
    if (own_buffers) return B2_OK;          // the segment sums follow on the tail stream (aggregate_segments)
    k_g2_segment_sum<<<n_seg, 32, 0, s>>>((const uint32_t*)aff.p, (const uint8_t*)st.p, d_seg_off, n_seg, (uint32_t*)V.sumjac.p, d_seg_status, n_sig, ctx->d_guard);
    CKL(ctx);
    return B2_OK;
}
static int aggregate_segments(b2_ctx* ctx, vslot& V, const uint32_t* d_seg_off, uint32_t n_seg, uint64_t n_sig, int32_t* d_seg_status, cudaStream_t t) {
    k_g2_segment_sum<<<n_seg, 32, 0, t>>>((const uint32_t*)V.g2aff.p, (const uint8_t*)V.g2st.p, d_seg_off, n_seg, (uint32_t*)V.sumjac.p, d_seg_status, n_sig,
                                           ctx->d_guard);
    CKL(ctx);
    return B2_OK;
}
static int aggregate_finish(b2_ctx* ctx, vslot& V, uint32_t n_seg, uint8_t* d_out96, const int32_t* d_seg_status, bool handoff, cudaStream_t s,
                            unsigned tb = 32) {
    int rc;
    if (handoff && ((rc = ensure(ctx, V.saff, (size_t)n_seg * 192)) || (rc = ensure(ctx, V.sflag, n_seg)))) return rc;
    k_g2_finish<<<blocks_for(n_seg, tb), tb, 0, s>>>((const uint32_t*)V.sumjac.p, d_seg_status, n_seg, d_out96,
                                                    handoff ? (uint32_t*)V.saff.p : nullptr, handoff ? (uint8_t*)V.sflag.p : nullptr);
    CKL(ctx);
    return B2_OK;
}

static int check_aggregate(b2_ctx* ctx, const uint8_t* sig96, const uint32_t* seg_off, uint32_t n_seg, uint64_t n_sig, const uint8_t* out96,
                           const int32_t* seg_status) {
    REQUIRE(ctx && seg_off && out96 && seg_status && n_seg > 0, "aggregate: bad arguments");
    return n_sig == 0 || sig96 ? B2_OK : reject(ctx, "aggregate", "null signatures");
}
int b2_aggregate_dev(b2_ctx* ctx, const uint8_t* d_sig96, const uint32_t* d_seg_off, uint32_t n_seg, uint64_t n_sig, uint8_t* d_out96,
                     int32_t* d_seg_status, void* stream) {
    B2_NVTX;
    int rc;
    if ((rc = check_aggregate(ctx, d_sig96, d_seg_off, n_seg, n_sig, d_out96, d_seg_status))) return rc;
    CK(cudaSetDevice(ctx->device));
    if ((rc = aggregate_front(ctx, ctx->slot[0], d_sig96, d_seg_off, n_seg, n_sig, d_seg_status, (cudaStream_t)stream))) return rc;
    return aggregate_finish(ctx, ctx->slot[0], n_seg, d_out96, d_seg_status, false, (cudaStream_t)stream);
}

int b2_aggregate(b2_ctx* ctx, const uint8_t* sig96, const uint32_t* seg_off, uint32_t n_seg, uint8_t* out96, int32_t* seg_status) {
    B2_NVTX;
    REQUIRE(ctx && seg_off, "aggregate: bad arguments");
    int rc;
    if ((rc = check_offsets(ctx, seg_off, n_seg, "aggregate", "seg_off"))) return rc;
    const uint64_t n_sig = seg_off[n_seg];
    if ((rc = check_aggregate(ctx, sig96, seg_off, n_seg, n_sig, out96, seg_status))) return rc;
    CK(cudaSetDevice(ctx->device));
    staging st(ctx);
    const uint8_t* dsig = st.in(sig96, n_sig * 96, 16);
    const uint32_t* doff = st.in(seg_off, (size_t)n_seg + 1);
    uint8_t* d96 = st.out(out96, (size_t)n_seg * 96);
    int32_t* dst = st.out(seg_status, n_seg);
    if ((rc = st.rc) || (rc = b2_aggregate_dev(ctx, dsig, doff, n_seg, n_sig, d96, dst, ctx->s_main))) return rc;
    return st.finish();
}

// ------------------------------------------------------------------------------------------ FastAggregateVerify
// Verification pipeline on three streams.  Nothing on the two side streams depends on the signatures:
//   aux0: K4 hash-to-G2
//   aux1: K2 pubkey gather+aggregate (or the explicit-key variant), then [after aux0] the Miller loop e(PK_agg, H(m))
//   main: signature decompression + subgroup check, Miller loop e(-g1, sig), [join aux1] final exponentiation.
// verify_fork() enqueues the side work forked from the *current* position of the caller's stream, verify_main()
// the signature half.  All intermediate buffers and events live in a `vslot`; the pipelined epoch API alternates
// between two slots so that the latency-bound tail of epoch k overlaps with the signature decompression of epoch k+1.
struct pk_source {
    const uint32_t *d_members, *d_off;
    const uint8_t* d_bits;
    uint32_t bits_stride;
    const uint8_t* d_pk48;      // explicit-key form when non-null (d_off = pk offsets)
    uint64_t n_pk;
    const uint32_t* d_committee;      // sync-committee form when non-null: block i = committee d_committee[i] of ctx->sync, bit row d_bits + i * ceil(size / 8)
    uint8_t* d_pk48_out;              // sync-committee form: compressed aggregate key per block (may be null)
    // split form when n_chunks > 0: aggregate i = the n_chunks aggregates i * n_chunks .. of the committee form (d_members, d_off, d_bits,
    // bits_stride), each summed by a warp of its own into d_part_jac / d_part_st, then added up (k_bae_pk_combine)
    uint32_t n_chunks;
    uint32_t* d_part_jac;
    uint8_t* d_part_st;
};
// Two forms of K5/K6.  `team`: three lanes per pairing -- shortest critical path, used when the caller waits for the result
// (synchronous entry points).  Thread-per-item: 2.7x longer, but ~40 % fewer warp instructions in total -- used by the pipelined
// epoch API, where the latency hides behind the next epoch's decompression and only the stolen multiply-pipe time counts.
static inline bool use_team(const b2_ctx* ctx, bool team) { return ctx->pairing_form == 0 ? team : ctx->pairing_form == 1; }
static int launch_miller(b2_ctx* ctx, vslot& V, uint32_t n_agg, int mode, bool team, cudaStream_t s) {
    team = use_team(ctx, team);
    if (team) {
        k_miller_team<<<blocks_for(n_agg, B2_TEAMS_PER_WARP), 32, B2_TEAM_SMEM, s>>>(
            (const uint32_t*)V.pkjac.p, (const uint8_t*)V.pkst.p, (const uint32_t*)V.haff.p, (const uint8_t*)V.hflag.p, (const uint32_t*)V.saff.p,
            (const uint8_t*)V.sflag.p, n_agg, (uint32_t*)V.f.p, mode);
    } else {
        k_miller<<<blocks_for(n_agg, ctx->tail_block), ctx->tail_block, 0, s>>>((const uint32_t*)V.pkjac.p, (const uint8_t*)V.pkst.p, (const uint32_t*)V.haff.p,
                                                      (const uint8_t*)V.hflag.p, (const uint32_t*)V.saff.p, (const uint8_t*)V.sflag.p, n_agg,
                                                      (uint32_t*)V.f.p, mode);
    }
    CKL(ctx);
    return B2_OK;
}
static int launch_final(b2_ctx* ctx, vslot& V, uint32_t n_agg, uint8_t* d_ok, bool team, cudaStream_t s) {
    team = use_team(ctx, team);
    if (team) {
        k_final_team<<<blocks_for(n_agg, B2_TEAMS_PER_WARP), 32, B2_TEAM_SMEM, s>>>((const uint32_t*)V.f.p, (const uint8_t*)V.pkst.p,
                                                                                  (const uint8_t*)V.sflag.p, n_agg, d_ok);
    } else {
        k_final_verdict<<<blocks_for(n_agg, ctx->tail_block), ctx->tail_block, 0, s>>>((const uint32_t*)V.f.p, (const uint8_t*)V.pkst.p, (const uint8_t*)V.sflag.p, n_agg, d_ok);
    }
    CKL(ctx);
    return B2_OK;
}
static int verify_fork(b2_ctx* ctx, vslot& V, const pk_source& P, const uint8_t* d_msg32, uint32_t n_agg, cudaStream_t s, bool team = true) {
    int rc;
    if ((rc = ensure(ctx, V.haff, (size_t)n_agg * 192)) || (rc = ensure(ctx, V.hflag, n_agg)) || (rc = ensure(ctx, V.saff, (size_t)n_agg * 192)) ||
        (rc = ensure(ctx, V.sflag, n_agg)) || (rc = ensure(ctx, V.f, (size_t)n_agg * 2 * 576)) || (rc = ensure(ctx, V.pkjac, (size_t)n_agg * 144)) ||
        (rc = ensure(ctx, V.pkst, n_agg)))
        return rc;
    if (P.d_pk48 && ((rc = ensure(ctx, ctx->sc_rec, P.n_pk * 96 + 16)) || (rc = ensure(ctx, ctx->sc_val, P.n_pk + 16)))) return rc;
    CK(cudaEventRecord(V.ev_fork, s));
    CK(cudaStreamWaitEvent(V.s_aux[0], V.ev_fork, 0));
    CK(cudaStreamWaitEvent(V.s_aux[1], V.ev_fork, 0));
    const unsigned tb = team ? 32u : ctx->tail_block;
    k_hash_to_g2<<<blocks_for(2ull * n_agg, tb), tb, 0, V.s_aux[0]>>>(d_msg32, n_agg, (uint32_t*)V.haff.p, (uint8_t*)V.hflag.p);
    CKL(ctx);
    CK(cudaEventRecord(V.ev_join0, V.s_aux[0]));
    if (P.d_pk48) {
        if (P.n_pk) {
            k_g1_decompress_validate<<<blocks_for(P.n_pk, 128), 128, 0, V.s_aux[1]>>>(P.d_pk48, P.n_pk, (uint32_t*)ctx->sc_rec.p, (uint8_t*)ctx->sc_val.p);
            CKL(ctx);
        }
        k_g1_segment_sum<<<n_agg, 128, 0, V.s_aux[1]>>>((const uint32_t*)ctx->sc_rec.p, (const uint8_t*)ctx->sc_val.p, P.d_off, n_agg,
                                                          (uint32_t*)V.pkjac.p, (uint8_t*)V.pkst.p);
        CKL(ctx);
    } else if (P.d_committee) {
        const sync_tables& T = ctx->sync;
        k_sync_aggregate_pk<<<blocks_for(n_agg, B2_SYNC_WARPS), 32 * B2_SYNC_WARPS, 0, V.s_aux[1]>>>(T.records, T.valid, T.sum, T.size, T.n, P.d_committee,
                                                                                                    P.d_bits, n_agg, V.pkjac, V.pkst, ctx->d_guard);
        CKL(ctx);
        if (P.d_pk48_out) {
            k_g1_compress<<<blocks_for(n_agg, 64), 64, 0, V.s_aux[1]>>>(V.pkjac, n_agg, P.d_pk48_out);
            CKL(ctx);
        }
    } else if (P.n_chunks) {
        const uint64_t n_part = (uint64_t)n_agg * P.n_chunks;
        k_g1_gather_tma<false><<<blocks_for(n_part, 4), 128, 4 * sizeof(gather_ws), V.s_aux[1]>>>(ctx->reg.records, P.d_members, P.d_off, P.d_bits,
                                                                                              P.bits_stride, (uint32_t)n_part, P.d_part_jac,
                                                                                              P.d_part_st, ctx->n_val, ctx->d_guard, nullptr);
        CKL(ctx);
        k_bae_pk_combine<<<blocks_for((uint64_t)n_agg * 32, 128), 128, 0, V.s_aux[1]>>>(P.d_part_jac, P.d_part_st, P.n_chunks, n_agg, V.pkjac, V.pkst);
        CKL(ctx);
    } else {
        // one block per aggregate.  128 threads when the caller waits; ONE WARP under the epoch pipeline: the 5-round shuffle tree costs
        // every warp 80 Fp multiplications whatever its share of the 512 records, so 4 warps spend 2.1x the multiply-pipe time of one
        const unsigned k2_block = team ? 128u : ctx->k2_block;
        if ((rc = launch_k2(ctx, P.d_members, P.d_off, P.d_bits, P.bits_stride, n_agg, (uint32_t*)V.pkjac.p, (uint8_t*)V.pkst.p, team ? 4u : 1u, k2_block,
                            V.s_aux[1])))
            return rc;
    }
    if (ctx->verify_mode == 1) {
        // RLC: the pubkey-side Miller loop runs on [r_i] PK_i (thread-per-aggregate kernels: this mode trades latency for work)
        const uint32_t n_groups = blocks_for(n_agg, B2_RLC_GROUP);
        if ((rc = ensure(ctx, V.pkjac_r, (size_t)n_agg * 144)) || (rc = ensure(ctx, V.rscal, (size_t)n_agg * 8)) || (rc = ensure(ctx, V.sg_aff, (size_t)n_groups * 192)) ||
            (rc = ensure(ctx, V.sg_flag, n_groups)) || (rc = ensure(ctx, V.f_g, (size_t)n_groups * 2 * 576)) || (rc = ensure(ctx, V.gpass, n_groups)))
            return rc;
        k_rlc_pk<<<blocks_for(n_agg, ctx->tail_block), ctx->tail_block, 0, V.s_aux[1]>>>(ctx->d_rlc_seed, d_msg32, (const uint32_t*)V.pkjac.p, (const uint8_t*)V.pkst.p,
                                                                                        n_agg, (unsigned long long*)V.rscal.p, (uint32_t*)V.pkjac_r.p);
        CKL(ctx);
        CK(cudaStreamWaitEvent(V.s_aux[1], V.ev_join0, 0));
        k_miller<<<blocks_for(n_agg, ctx->tail_block), ctx->tail_block, 0, V.s_aux[1]>>>((const uint32_t*)V.pkjac_r.p, (const uint8_t*)V.pkst.p, (const uint32_t*)V.haff.p,
                                                                                        (const uint8_t*)V.hflag.p, nullptr, nullptr, n_agg, (uint32_t*)V.f.p, 1);
        CKL(ctx);
        CK(cudaEventRecord(V.ev_join1, V.s_aux[1]));
        return B2_OK;
    }
    CK(cudaStreamWaitEvent(V.s_aux[1], V.ev_join0, 0));
    if ((rc = launch_miller(ctx, V, n_agg, 1, team, V.s_aux[1]))) return rc;
    CK(cudaEventRecord(V.ev_join1, V.s_aux[1]));
    return B2_OK;
}
// RLC batch mode, signature half + verdicts (V.saff / V.sflag hold the affine, subgroup-checked aggregate signatures)
static int verify_main_rlc(b2_ctx* ctx, vslot& V, uint32_t n_agg, uint8_t* d_ok, cudaStream_t s) {
    const uint32_t n_groups = blocks_for(n_agg, B2_RLC_GROUP);
    const unsigned tb = ctx->tail_block;
    const uint8_t *pkst = (const uint8_t*)V.pkst.p, *sflag = (const uint8_t*)V.sflag.p;
    k_rlc_sig<<<n_groups, 32, 0, s>>>((const uint32_t*)V.saff.p, sflag, pkst, (const unsigned long long*)V.rscal.p, n_agg, (uint32_t*)V.sg_aff.p, (uint8_t*)V.sg_flag.p);
    CKL(ctx);
    // e(-g1, sum [r_i] S_i) per group
    k_miller<<<blocks_for(n_groups, tb), tb, 0, s>>>(nullptr, nullptr, nullptr, nullptr, (const uint32_t*)V.sg_aff.p, (const uint8_t*)V.sg_flag.p, n_groups, (uint32_t*)V.f_g.p, 2);
    CKL(ctx);
    CK(cudaStreamWaitEvent(s, V.ev_join1, 0));
    k_rlc_final<<<blocks_for(n_groups, 32), 32, 0, s>>>((const uint32_t*)V.f.p, (const uint32_t*)V.f_g.p, pkst, sflag, n_agg, n_groups, (uint8_t*)V.gpass.p);
    CKL(ctx);
    k_rlc_verdict<<<blocks_for(n_agg, 128), 128, 0, s>>>(pkst, sflag, (const uint8_t*)V.gpass.p, n_agg, d_ok);
    CKL(ctx);
    // fallback: the members of a failed group, aggregate by aggregate (threads of passed groups exit at once)
    k_miller<<<blocks_for(2 * n_agg, tb), tb, 0, s>>>((const uint32_t*)V.pkjac.p, pkst, (const uint32_t*)V.haff.p, (const uint8_t*)V.hflag.p, (const uint32_t*)V.saff.p, sflag,
                                                       n_agg, (uint32_t*)V.f.p, 0, (const uint8_t*)V.gpass.p, B2_RLC_GROUP);
    CKL(ctx);
    k_final_verdict<<<blocks_for(n_agg, tb), tb, 0, s>>>((const uint32_t*)V.f.p, pkst, sflag, n_agg, d_ok, (const uint8_t*)V.gpass.p, B2_RLC_GROUP);
    CKL(ctx);
    return B2_OK;
}
// d_sig96 == nullptr: the signature points are already in V.saff / V.sflag (handed over by aggregate_finish)
static int verify_main(b2_ctx* ctx, vslot& V, const uint8_t* d_sig96, uint32_t n_agg, uint8_t* d_ok, cudaStream_t s, bool team = true) {
    int rc;
    if (d_sig96) {
        k_sig_prepare<<<blocks_for(n_agg, 32), 32, 0, s>>>(d_sig96, n_agg, (uint32_t*)V.saff.p, (uint8_t*)V.sflag.p);
        CKL(ctx);
    }
    if (ctx->verify_mode == 1) return verify_main_rlc(ctx, V, n_agg, d_ok, s);
    if ((rc = launch_miller(ctx, V, n_agg, 2, team, s))) return rc;
    CK(cudaStreamWaitEvent(s, V.ev_join1, 0));
    return launch_final(ctx, V, n_agg, d_ok, team, s);
}

static int check_fast_aggregate_verify(b2_ctx* ctx, const void* members, const void* off, const void* bits, uint32_t bits_stride, const void* msg32,
                                       const void* sig96, uint32_t n_agg, const void* ok_out) {
    REQUIRE(ctx && members && off && bits && msg32 && sig96 && ok_out && n_agg > 0 && bits_stride > 0, "fast_aggregate_verify: bad arguments");
    return ctx->n_val > 0 ? B2_OK : reject(ctx, "fast_aggregate_verify", "registry not loaded");
}
int b2_fast_aggregate_verify_dev(b2_ctx* ctx, const uint32_t* d_members, const uint32_t* d_off, const uint8_t* d_bits, uint32_t bits_stride,
                                 const uint8_t* d_msg32, const uint8_t* d_sig96, uint32_t n_agg, uint8_t* d_ok_out, void* stream) {
    B2_NVTX;
    int rc;
    if ((rc = check_fast_aggregate_verify(ctx, d_members, d_off, d_bits, bits_stride, d_msg32, d_sig96, n_agg, d_ok_out))) return rc;
    CK(cudaSetDevice(ctx->device));
    cudaStream_t s = (cudaStream_t)stream;
    pk_source P = {d_members, d_off, d_bits, bits_stride, nullptr, 0};
    if ((rc = verify_fork(ctx, ctx->slot[0], P, d_msg32, n_agg, s))) return rc;
    return verify_main(ctx, ctx->slot[0], d_sig96, n_agg, d_ok_out, s);
}

// ---- one epoch for the validators of this rank: per-committee bls.Aggregate of the individual signatures,
// FastAggregateVerify of the aggregates, update_latest_messages for the accepted ones.
//   epoch_start: fork the signature-independent half (hash, pubkey aggregation, first Miller loop) on the side streams,
//                then decompress + segment-sum the signatures on the caller's stream (the grid-filling part);
//   epoch_tail : inversion/compress + subgroup check, second Miller loop, final exponentiation, LMD update -- latency-
//                bound work on few SMs; on `tail_stream` (the caller's own stream, or the context's tail stream so that
//                it overlaps with the next epoch's epoch_start in the other slot).
static int epoch_start(b2_ctx* ctx, int slot, const uint8_t* d_sig96, const uint32_t* d_members, const uint32_t* d_off, const uint8_t* d_bits,
                       uint32_t bits_stride, const uint8_t* d_msg32, uint32_t n_agg, uint64_t n_sig, int32_t* d_agg_status, cudaStream_t s, bool team,
                       bool own_buffers = false) {
    vslot& V = ctx->slot[slot];
    int rc;
    CK(cudaStreamWaitEvent(s, V.ev_tail_done, 0));      // the slot's previous user (B2_EPOCH_SLOTS-or-fewer epochs ago) must have drained
    pk_source P = {d_members, d_off, d_bits, bits_stride, nullptr, 0};
    if ((rc = verify_fork(ctx, V, P, d_msg32, n_agg, s, team))) return rc;
    V.segsum_pending = own_buffers;
    V.n_sig_tail = n_sig;
    cudaStream_t sd = s;
    const bool few_waves = n_sig < (uint64_t)6 * ctx->n_sm * 4 * ctx->dec_block;
    if (own_buffers && (ctx->dec_alternate == 1 || (ctx->dec_alternate < 0 && few_waves))) {      // the slot's own point buffer makes this legal
        sd = ctx->s_dec[ctx->dec_turn++ % ctx->n_dec_streams];
        CK(cudaEventRecord(V.ev_in, s));                // inputs ready, slot drained
        CK(cudaStreamWaitEvent(sd, V.ev_in, 0));
    }
    if ((rc = aggregate_front(ctx, V, d_sig96, d_off, n_agg, n_sig, d_agg_status, sd, own_buffers))) return rc;
    CK(cudaEventRecord(V.ev_seg, sd));
    return B2_OK;
}
static int epoch_tail(b2_ctx* ctx, int slot, const uint32_t* d_members, const uint32_t* d_off, const uint8_t* d_bits, uint32_t bits_stride,
                      const uint64_t* d_target_epoch, const uint32_t* d_block_idx, uint32_t n_agg, uint8_t* d_agg_sig96, int32_t* d_agg_status,
                      uint8_t* d_ok_out, cudaStream_t t, bool team) {
    vslot& V = ctx->slot[slot];
    int rc;
    CK(cudaStreamWaitEvent(t, V.ev_seg, 0));
    if (V.segsum_pending) {
        if ((rc = aggregate_segments(ctx, V, d_off, n_agg, V.n_sig_tail, d_agg_status, t))) return rc;
        V.segsum_pending = false;
    }
    if ((rc = aggregate_finish(ctx, V, n_agg, d_agg_sig96, d_agg_status, true, t, team ? 32u : ctx->tail_block))) return rc;
    if ((rc = verify_main(ctx, V, nullptr, n_agg, d_ok_out, t, team))) return rc;
    if (d_target_epoch) {
        CK(cudaStreamWaitEvent(t, ctx->ev_votes_done, 0));  // do not move the LMD table under a vote scatter that is still reading it
        CK(cudaStreamWaitEvent(t, ctx->ev_lmd_done, 0));    // latest messages are applied in epoch order even when tails overlap
        CK(cudaStreamWaitEvent(t, ctx->ev_equiv_done, 0));  // ... and skip every validator the epochs before this one were found to equivocate
        if ((rc = b2_latest_messages_update_dev(ctx, d_members, d_off, d_bits, bits_stride, d_target_epoch, d_block_idx, d_ok_out, n_agg, t))) return rc;
        CK(cudaEventRecord(ctx->ev_lmd_done, t));
    }   // else: the caller applies update_latest_messages itself, after exchanging the verdicts of all ranks (sharded epoch)
    CK(cudaEventRecord(V.ev_tail_done, t));
    return B2_OK;
}

int b2_epoch_dev(b2_ctx* ctx, const uint8_t* d_sig96, const uint32_t* d_members, const uint32_t* d_off, const uint8_t* d_bits,
                 uint32_t bits_stride, const uint8_t* d_msg32, const uint64_t* d_target_epoch, const uint32_t* d_block_idx, uint32_t n_agg,
                 uint64_t n_sig, uint8_t* d_agg_sig96, int32_t* d_agg_status, uint8_t* d_ok_out, void* stream) {
    B2_NVTX;
    REQUIRE(ctx && d_sig96 && d_members && d_off && d_bits && d_msg32 && (!d_target_epoch == !d_block_idx) && d_agg_sig96 && d_agg_status && d_ok_out &&
                n_agg > 0 && bits_stride > 0, "epoch_dev: bad arguments");
    REQUIRE(ctx->n_val > 0, "epoch_dev: registry not loaded");
    CK(cudaSetDevice(ctx->device));
    cudaStream_t s = (cudaStream_t)stream;
    int rc;
    if ((rc = epoch_start(ctx, 0, d_sig96, d_members, d_off, d_bits, bits_stride, d_msg32, n_agg, n_sig, d_agg_status, s, true))) return rc;
    return epoch_tail(ctx, 0, d_members, d_off, d_bits, bits_stride, d_target_epoch, d_block_idx, n_agg, d_agg_sig96, d_agg_status, d_ok_out, s, true);
}

// Pipelined form: per epoch k, slot = k mod depth (depth <= B2_EPOCH_SLOTS): start(slot) on the caller's stream, tail(slot) on the
// slot's own high-priority stream, then the fork choice of the epoch on any stream after b2_epoch_wait_dev(slot, stream).  Tails of
// consecutive epochs overlap each other and the following decompressions; latest messages are still applied in epoch order.
int b2_epoch_start_dev(b2_ctx* ctx, int slot, const uint8_t* d_sig96, const uint32_t* d_members, const uint32_t* d_off, const uint8_t* d_bits,
                       uint32_t bits_stride, const uint8_t* d_msg32, uint32_t n_agg, uint64_t n_sig, int32_t* d_agg_status, void* stream) {
    B2_NVTX;
    REQUIRE(ctx && slot >= 0 && slot < B2_EPOCH_SLOTS && d_sig96 && d_members && d_off && d_bits && d_msg32 && d_agg_status && n_agg > 0 && bits_stride > 0,
            "epoch_start_dev: bad arguments");
    REQUIRE(ctx->n_val > 0, "epoch_start_dev: registry not loaded");
    CK(cudaSetDevice(ctx->device));
    return epoch_start(ctx, slot, d_sig96, d_members, d_off, d_bits, bits_stride, d_msg32, n_agg, n_sig, d_agg_status, (cudaStream_t)stream,
                       ctx->epoch_team, true);
}
int b2_epoch_tail_dev(b2_ctx* ctx, int slot, const uint32_t* d_members, const uint32_t* d_off, const uint8_t* d_bits, uint32_t bits_stride,
                      const uint64_t* d_target_epoch, const uint32_t* d_block_idx, uint32_t n_agg, uint8_t* d_agg_sig96, int32_t* d_agg_status,
                      uint8_t* d_ok_out) {
    B2_NVTX;
    REQUIRE(ctx && slot >= 0 && slot < B2_EPOCH_SLOTS && d_members && d_off && d_bits && (!d_target_epoch == !d_block_idx) && d_agg_sig96 && d_agg_status && d_ok_out &&
                n_agg > 0 && bits_stride > 0, "epoch_tail_dev: bad arguments");
    CK(cudaSetDevice(ctx->device));
    return epoch_tail(ctx, slot, d_members, d_off, d_bits, bits_stride, d_target_epoch, d_block_idx, n_agg, d_agg_sig96, d_agg_status, d_ok_out,
                      ctx->slot[slot].s_tail, ctx->epoch_team);
}
// Vote form of the epoch (votes.cuh): group the members and signatures by vote so that the epoch entry points run one segment per vote.
int b2_votes_group_dev(b2_ctx* ctx, const uint32_t* d_vote, const uint32_t* d_vote_off, uint32_t n_votes, const uint32_t* d_members, const uint32_t* d_off,
                       uint32_t n_committees, uint64_t n_sig, uint32_t bits_stride, const uint8_t* d_sig96, uint32_t c_begin, uint32_t c_end,
                       uint8_t* d_sig96_out, uint32_t* d_members_out, uint32_t* d_pos_out, uint32_t* d_seg_off, uint32_t* d_seg_off_loc,
                       uint8_t* d_bits_out, uint8_t* d_agg_bits_out, void* stream) {
    B2_NVTX;
    REQUIRE(ctx && d_vote && d_vote_off && d_members && d_off && d_sig96 && d_sig96_out && d_members_out && d_pos_out && d_seg_off && d_bits_out &&
                d_agg_bits_out && n_votes > 0 && n_committees > 0 && n_sig < (1ull << 32) && bits_stride > 0 && bits_stride <= 256 &&
                c_begin < c_end && c_end <= n_committees,
            "votes_group_dev: bad arguments");
    CK(cudaSetDevice(ctx->device));
    vote_group_args A = {d_vote, d_vote_off, d_off, d_members, n_committees, n_votes, bits_stride, n_sig, d_sig96, c_begin, c_end, d_sig96_out,
                    d_members_out, d_pos_out, d_seg_off, d_seg_off_loc, d_bits_out, d_agg_bits_out, ctx->d_guard};
    k_votes_group<<<n_committees, VOTES_THREADS, 0, (cudaStream_t)stream>>>(A);
    CKL(ctx);
    return B2_OK;
}
int b2_votes_empty_dev(b2_ctx* ctx, const uint8_t* d_bits, uint32_t bits_stride, uint32_t n_votes, uint8_t* d_agg_sig96, int32_t* d_agg_status, void* stream) {
    B2_NVTX;
    REQUIRE(ctx && d_bits && d_agg_sig96 && n_votes > 0 && bits_stride > 0, "votes_empty_dev: bad arguments");
    CK(cudaSetDevice(ctx->device));
    k_votes_empty<<<blocks_for((uint64_t)n_votes * 24, 256), 256, 0, (cudaStream_t)stream>>>(d_bits, bits_stride, n_votes, d_agg_sig96, d_agg_status);
    CKL(ctx);
    return B2_OK;
}
int b2_epoch_set_pairing_form(b2_ctx* ctx, int form) {
    B2_NVTX;
    REQUIRE(ctx && (form == 0 || form == 1), "epoch_set_pairing_form: bad arguments");
    ctx->epoch_team = form == 1;
    return B2_OK;
}
int b2_epoch_wait_dev(b2_ctx* ctx, int slot, void* stream) {
    B2_NVTX;
    REQUIRE(ctx && slot >= 0 && slot < B2_EPOCH_SLOTS, "epoch_wait_dev: bad arguments");
    CK(cudaSetDevice(ctx->device));
    CK(cudaStreamWaitEvent((cudaStream_t)stream, ctx->slot[slot].ev_tail_done, 0));
    return B2_OK;
}

int b2_fast_aggregate_verify(b2_ctx* ctx, const uint32_t* members, const uint32_t* off, const uint8_t* bits, uint32_t bits_stride,
                             const uint8_t* msg32, const uint8_t* sig96, uint32_t n_agg, uint8_t* ok_out) {
    B2_NVTX;
    int rc;
    if ((rc = check_fast_aggregate_verify(ctx, members, off, bits, bits_stride, msg32, sig96, n_agg, ok_out)) ||
        (rc = check_batch(ctx, members, off, bits_stride, n_agg, ctx->n_val, "fast_aggregate_verify")))
        return rc;
    CK(cudaSetDevice(ctx->device));
    staging st(ctx);
    const uint32_t* dm = st.in(members, off[n_agg], 4);
    const uint32_t* dof = st.in(off, (size_t)n_agg + 1);
    const uint8_t* db = st.in(bits, (size_t)n_agg * bits_stride, 16);
    const uint8_t* dsig = st.in(sig96, (size_t)n_agg * 96);
    const uint8_t* dmsg = st.in(msg32, (size_t)n_agg * 32);
    uint8_t* dok = st.out(ok_out, n_agg);
    if ((rc = st.rc) || (rc = b2_fast_aggregate_verify_dev(ctx, dm, dof, db, bits_stride, dmsg, dsig, n_agg, dok, ctx->s_main))) return rc;
    return st.finish();
}

int b2_fast_aggregate_verify_pks(b2_ctx* ctx, const uint8_t* pk48, const uint32_t* pk_off, const uint8_t* msg32, const uint8_t* sig96,
                                 uint32_t n_agg, uint8_t* ok_out) {
    B2_NVTX;
    REQUIRE(ctx && pk_off && msg32 && sig96 && ok_out && n_agg > 0, "fast_aggregate_verify_pks: bad arguments");
    int rc;
    if ((rc = check_offsets(ctx, pk_off, n_agg, "fast_aggregate_verify_pks", "pk_off"))) return rc;
    const uint64_t n_pk = pk_off[n_agg];
    REQUIRE(n_pk == 0 || pk48, "null pubkeys");
    CK(cudaSetDevice(ctx->device));
    cudaStream_t s = ctx->s_main;
    if ((rc = ensure(ctx, ctx->sc_rec, n_pk * 96 + 16)) || (rc = ensure(ctx, ctx->sc_val, n_pk + 16)) ||
        (rc = ensure(ctx, ctx->sc_pkjac, (size_t)n_agg * 144)) || (rc = ensure(ctx, ctx->sc_pkst, n_agg)))
        return rc;
    staging st(ctx);
    const uint8_t* dpk = st.in(pk48, n_pk * 48, 16);
    const uint32_t* dof = st.in(pk_off, (size_t)n_agg + 1);
    const uint8_t* dsig = st.in(sig96, (size_t)n_agg * 96);
    const uint8_t* dmsg = st.in(msg32, (size_t)n_agg * 32);
    uint8_t* dok = st.out(ok_out, n_agg);
    pk_source P = {nullptr, dof, nullptr, 0, dpk, n_pk};
    if ((rc = st.rc) || (rc = verify_fork(ctx, ctx->slot[0], P, dmsg, n_agg, s)) || (rc = verify_main(ctx, ctx->slot[0], dsig, n_agg, dok, s))) return rc;
    return st.finish();
}

// ------------------------------------------------------------------------------------------ AggregateVerify / AggregatePKs
// Keys by registry index (d_signer) or explicit (d_pk48, decoded + KeyValidated here).  Hashing and key decoding fork onto the
// context's AggregateVerify side streams; signature preparation, the per-item Miller loops and the per-set final exponentiations
// run on `s`.  The grid covers n_pairs + n_sets items whatever the offsets say; k_av_check makes the kernels that follow skip the
// whole batch when the offsets are malformed.
static int aggregate_verify_enqueue(b2_ctx* ctx, const uint32_t* d_signer, const uint8_t* d_pk48, const uint8_t* d_msg32, const uint32_t* d_pair_off,
                                    uint64_t n_pairs, const uint8_t* d_sig96, uint32_t n_sets, uint8_t* d_ok, cudaStream_t s) {
    const unsigned n_blocks = blocks_for(n_pairs + n_sets, B2_AV_BLOCK);
    const size_t n_slots = (size_t)n_sets + n_blocks;
    int rc;
    if ((rc = ensure(ctx, ctx->sc_haff, n_pairs * 192 + 16)) || (rc = ensure(ctx, ctx->sc_hflag, n_pairs + 16)) ||
        (rc = ensure(ctx, ctx->sc_av_saff, (size_t)n_sets * 192)) || (rc = ensure(ctx, ctx->sc_av_sflag, n_sets)) ||
        (rc = ensure(ctx, ctx->sc_av_f, n_slots * 576)) || (rc = ensure(ctx, ctx->sc_av_st, n_slots * 4)) || (rc = ensure(ctx, ctx->sc_av_bad, 4)))
        return rc;
    if (d_pk48 && ((rc = ensure(ctx, ctx->sc_rec, n_pairs * 96 + 16)) || (rc = ensure(ctx, ctx->sc_val, n_pairs + 16)))) return rc;
    uint32_t* bad_row = ctx->sc_av_bad;
    CK(cudaMemsetAsync(bad_row, 0, 4, s));
    k_av_check<<<blocks_for(n_sets, 128), 128, 0, s>>>(d_pair_off, n_sets, n_pairs, bad_row, ctx->d_guard);
    CKL(ctx);
    if (n_pairs) {
        CK(cudaEventRecord(ctx->ev_av[0], s));
        CK(cudaStreamWaitEvent(ctx->s_av[0], ctx->ev_av[0], 0));
        k_hash_to_g2<<<blocks_for(2 * n_pairs, 32), 32, 0, ctx->s_av[0]>>>(d_msg32, (uint32_t)n_pairs, ctx->sc_haff, ctx->sc_hflag);
        CKL(ctx);
        CK(cudaEventRecord(ctx->ev_av[1], ctx->s_av[0]));
        if (d_pk48) {
            CK(cudaStreamWaitEvent(ctx->s_av[1], ctx->ev_av[0], 0));
            k_g1_decompress_validate<<<blocks_for(n_pairs, 128), 128, 0, ctx->s_av[1]>>>(d_pk48, n_pairs, ctx->sc_rec, ctx->sc_val);
            CKL(ctx);
            CK(cudaEventRecord(ctx->ev_av[2], ctx->s_av[1]));
        }
    }
    k_sig_prepare<<<blocks_for(n_sets, 32), 32, 0, s>>>(d_sig96, n_sets, ctx->sc_av_saff, ctx->sc_av_sflag);
    CKL(ctx);
    if (n_pairs) {
        CK(cudaStreamWaitEvent(s, ctx->ev_av[1], 0));
        if (d_pk48) CK(cudaStreamWaitEvent(s, ctx->ev_av[2], 0));
    }
    const uint32_t* records = d_pk48 ? (const uint32_t*)ctx->sc_rec : (const uint32_t*)ctx->reg.records;
    const uint8_t* valid = d_pk48 ? (const uint8_t*)ctx->sc_val : (const uint8_t*)ctx->reg.valid;
    k_av_miller<<<n_blocks, B2_AV_BLOCK, 0, s>>>(d_pair_off, n_sets, d_signer, records, valid, d_pk48 ? n_pairs : ctx->n_val,
                                                 ctx->sc_haff, ctx->sc_hflag, ctx->sc_av_saff, ctx->sc_av_sflag, bad_row, ctx->sc_av_f, ctx->sc_av_st,
                                                 ctx->d_guard);
    CKL(ctx);
    k_av_final<<<blocks_for(n_sets, 32), 32, 0, s>>>(d_pair_off, n_sets, bad_row, ctx->sc_av_f, ctx->sc_av_st, d_ok);
    CKL(ctx);
    return B2_OK;
}

static int check_aggregate_verify(b2_ctx* ctx, const uint32_t* signer, const uint8_t* msg32, const uint32_t* pair_off, uint64_t n_pairs,
                                  const uint8_t* sig96, uint32_t n_sets, const uint8_t* ok_out) {
    REQUIRE(ctx && pair_off && sig96 && ok_out && n_sets > 0, "aggregate_verify: bad arguments");
    REQUIRE(n_pairs == 0 || (signer && msg32), "aggregate_verify: null signers or messages");
    REQUIRE(n_pairs + n_sets < (1ull << 32), "aggregate_verify: too many pairs");
    return ctx->n_val > 0 ? B2_OK : reject(ctx, "aggregate_verify", "registry not loaded");
}
int b2_aggregate_verify_dev(b2_ctx* ctx, const uint32_t* d_signer, const uint8_t* d_msg32, const uint32_t* d_pair_off, uint64_t n_pairs, const uint8_t* d_sig96,
                            uint32_t n_sets, uint8_t* d_ok_out, void* stream) {
    B2_NVTX;
    int rc;
    if ((rc = check_aggregate_verify(ctx, d_signer, d_msg32, d_pair_off, n_pairs, d_sig96, n_sets, d_ok_out))) return rc;
    CK(cudaSetDevice(ctx->device));
    return aggregate_verify_enqueue(ctx, d_signer, nullptr, d_msg32, d_pair_off, n_pairs, d_sig96, n_sets, d_ok_out, (cudaStream_t)stream);
}

int b2_aggregate_verify(b2_ctx* ctx, const uint32_t* signer, const uint8_t* msg32, const uint32_t* pair_off, const uint8_t* sig96, uint32_t n_sets,
                        uint8_t* ok_out) {
    B2_NVTX;
    REQUIRE(ctx && pair_off, "aggregate_verify: bad arguments");
    int rc;
    if ((rc = check_offsets(ctx, pair_off, n_sets, "aggregate_verify", "pair_off"))) return rc;
    const uint64_t n_pairs = pair_off[n_sets];
    if ((rc = check_aggregate_verify(ctx, signer, msg32, pair_off, n_pairs, sig96, n_sets, ok_out))) return rc;
    for (uint64_t i = 0; i < n_pairs; i++) REQUIRE(signer[i] < ctx->n_val, "aggregate_verify: signer index outside the registry");
    CK(cudaSetDevice(ctx->device));
    staging st(ctx);
    const uint32_t* dsigner = st.in(signer, n_pairs, 4);
    const uint8_t* dmsg = st.in(msg32, n_pairs * 32, 16);
    const uint32_t* doff = st.in(pair_off, (size_t)n_sets + 1);
    const uint8_t* dsig = st.in(sig96, (size_t)n_sets * 96);
    uint8_t* dok = st.out(ok_out, n_sets);
    if ((rc = st.rc) || (rc = aggregate_verify_enqueue(ctx, dsigner, nullptr, dmsg, doff, n_pairs, dsig, n_sets, dok, ctx->s_main))) return rc;
    return st.finish();
}

int b2_aggregate_verify_pks(b2_ctx* ctx, const uint8_t* pk48, const uint8_t* msg32, const uint32_t* pair_off, const uint8_t* sig96, uint32_t n_sets,
                            uint8_t* ok_out) {
    B2_NVTX;
    REQUIRE(ctx && pair_off && sig96 && ok_out && n_sets > 0, "aggregate_verify_pks: bad arguments");
    int rc;
    if ((rc = check_offsets(ctx, pair_off, n_sets, "aggregate_verify_pks", "pair_off"))) return rc;
    const uint64_t n_pairs = pair_off[n_sets];
    REQUIRE(n_pairs == 0 || (pk48 && msg32), "aggregate_verify_pks: null pubkeys or messages");
    REQUIRE(n_pairs + n_sets < (1ull << 32), "aggregate_verify_pks: too many pairs");
    CK(cudaSetDevice(ctx->device));
    staging st(ctx);
    const uint8_t* dpk = st.in(pk48, n_pairs * 48, 16);
    const uint8_t* dmsg = st.in(msg32, n_pairs * 32, 16);
    const uint32_t* doff = st.in(pair_off, (size_t)n_sets + 1);
    const uint8_t* dsig = st.in(sig96, (size_t)n_sets * 96);
    uint8_t* dok = st.out(ok_out, n_sets);
    if ((rc = st.rc) || (rc = aggregate_verify_enqueue(ctx, nullptr, dpk, dmsg, doff, n_pairs, dsig, n_sets, dok, ctx->s_main))) return rc;
    return st.finish();
}

// py_ecc _AggregatePKs, batched: decode + KeyValidate every key, per-segment sums (the status bits of b2_g1_aggregate), compress
int b2_aggregate_pks(b2_ctx* ctx, const uint8_t* pk48, const uint32_t* off, uint32_t n_seg, uint8_t* out48, uint8_t* status) {
    B2_NVTX;
    REQUIRE(ctx && off && out48 && status && n_seg > 0, "aggregate_pks: bad arguments");
    int rc;
    if ((rc = check_offsets(ctx, off, n_seg, "aggregate_pks"))) return rc;
    const uint64_t n_pk = off[n_seg];
    REQUIRE(n_pk == 0 || pk48, "aggregate_pks: null pubkeys");
    CK(cudaSetDevice(ctx->device));
    cudaStream_t s = ctx->s_main;
    staging st(ctx);
    const uint8_t* dpk = st.in(pk48, n_pk * 48, 16);
    const uint32_t* doff = st.in(off, (size_t)n_seg + 1);
    uint8_t* d48 = st.out(out48, (size_t)n_seg * 48);
    if ((rc = st.rc) || (rc = ensure(ctx, ctx->sc_rec, n_pk * 96 + 16)) || (rc = ensure(ctx, ctx->sc_val, n_pk + 16)) ||
        (rc = ensure(ctx, ctx->sc_pkjac, (size_t)n_seg * 144)) || (rc = ensure(ctx, ctx->sc_pkst, n_seg)))
        return rc;
    if (n_pk) {
        k_g1_decompress_validate<<<blocks_for(n_pk, 128), 128, 0, s>>>(dpk, n_pk, ctx->sc_rec, ctx->sc_val);
        CKL(ctx);
    }
    k_g1_segment_sum<<<n_seg, 128, 0, s>>>(ctx->sc_rec, ctx->sc_val, doff, n_seg, ctx->sc_pkjac, ctx->sc_pkst);
    CKL(ctx);
    k_g1_compress<<<blocks_for(n_seg, 64), 64, 0, s>>>(ctx->sc_pkjac, n_seg, d48);
    CKL(ctx);
    st.out(status, ctx->sc_pkst, n_seg);
    return st.finish();
}

// ------------------------------------------------------------------------------------------ sync committees (syncagg.cuh)
// Decode + KeyValidate every key and sum each committee's valid keys, into tables built aside: the loaded committees are replaced
// only once the new ones are complete.
int b2_sync_committee_load(b2_ctx* ctx, const uint8_t* pk48, uint32_t committee_size, uint32_t n_committees, uint8_t* valid_out) {
    B2_NVTX;
    REQUIRE(ctx && pk48 && committee_size > 0 && n_committees > 0, "sync_committee_load: bad arguments");
    REQUIRE(committee_size <= B2_SYNC_MAX_SIZE, "sync_committee_load: committee_size above the kernel's limit (1024)");
    const uint64_t n_pk = (uint64_t)committee_size * n_committees;
    REQUIRE(n_pk < (1ull << 32), "sync_committee_load: too many keys");
    CK(cudaSetDevice(ctx->device));
    sync_tables t;
    int rc;
    if ((rc = ensure(ctx, t.records, n_pk * 96)) || (rc = ensure(ctx, t.valid, n_pk)) || (rc = ensure(ctx, t.sum, (size_t)n_committees * 144)) ||
        (rc = ensure(ctx, t.sum_status, n_committees)))
        return rc;
    std::vector<uint32_t> off(n_committees + 1);
    for (uint32_t c = 0; c <= n_committees; c++) off[c] = c * committee_size;
    staging st(ctx);
    const uint8_t* dpk = st.in(pk48, n_pk * 48);
    const uint32_t* doff = st.in(off.data(), off.size());
    if (st.rc) return st.rc;
    cudaStream_t s = ctx->s_main;
    k_g1_decompress_validate<<<blocks_for(n_pk, 128), 128, 0, s>>>(dpk, n_pk, t.records, t.valid);
    CKL(ctx);
    k_g1_segment_sum<<<n_committees, 128, 0, s>>>(t.records, t.valid, doff, n_committees, t.sum, t.sum_status);
    CKL(ctx);
    if (valid_out) st.out(valid_out, t.valid, n_pk);
    if ((rc = st.finish())) return rc;
    t.size = committee_size;
    t.n = n_committees;
    ctx->sync = std::move(t);
    return B2_OK;
}

static int check_sync_aggregate_verify(b2_ctx* ctx, const void* committee_idx, const void* bits, const void* msg32, const void* sig96, uint32_t n,
                                       const void* ok_out) {
    REQUIRE(ctx && committee_idx && bits && msg32 && sig96 && ok_out && n > 0, "sync_aggregate_verify: bad arguments");
    return ctx->sync.n > 0 ? B2_OK : reject(ctx, "sync_aggregate_verify", "no sync committee loaded");
}
// eth_fast_aggregate_verify per block: the committee form of verify_fork (k_sync_aggregate_pk), the unchanged pairing half, then the
// empty-participation rule on the verdicts
int b2_sync_aggregate_verify_dev(b2_ctx* ctx, const uint32_t* d_committee_idx, const uint8_t* d_bits, const uint8_t* d_msg32, const uint8_t* d_sig96,
                                 uint32_t n, uint8_t* d_ok_out, uint8_t* d_pk48_out, void* stream) {
    B2_NVTX;
    int rc;
    if ((rc = check_sync_aggregate_verify(ctx, d_committee_idx, d_bits, d_msg32, d_sig96, n, d_ok_out))) return rc;
    CK(cudaSetDevice(ctx->device));
    cudaStream_t s = (cudaStream_t)stream;
    vslot& V = ctx->slot[0];
    pk_source P = {nullptr, nullptr, d_bits, 0, nullptr, 0, d_committee_idx, d_pk48_out};
    if ((rc = verify_fork(ctx, V, P, d_msg32, n, s)) || (rc = verify_main(ctx, V, d_sig96, n, d_ok_out, s))) return rc;
    k_sync_empty_verdict<<<blocks_for(n, 128), 128, 0, s>>>(V.pkst, d_sig96, n, d_ok_out);
    CKL(ctx);
    return B2_OK;
}

int b2_sync_aggregate_verify(b2_ctx* ctx, const uint32_t* committee_idx, const uint8_t* bits, const uint8_t* msg32, const uint8_t* sig96, uint32_t n,
                             uint8_t* ok_out, uint8_t* pk48_out) {
    B2_NVTX;
    int rc;
    if ((rc = check_sync_aggregate_verify(ctx, committee_idx, bits, msg32, sig96, n, ok_out))) return rc;
    for (uint32_t i = 0; i < n; i++) REQUIRE(committee_idx[i] < ctx->sync.n, "sync_aggregate_verify: committee index out of range");
    CK(cudaSetDevice(ctx->device));
    const size_t stride = (ctx->sync.size + 7) / 8;
    staging st(ctx);
    const uint32_t* dc = st.in(committee_idx, n);
    const uint8_t* db = st.in(bits, n * stride, 16);
    const uint8_t* dmsg = st.in(msg32, (size_t)n * 32);
    const uint8_t* dsig = st.in(sig96, (size_t)n * 96);
    uint8_t* dok = st.out(ok_out, n);
    uint8_t* d48 = pk48_out ? st.out(pk48_out, (size_t)n * 48) : nullptr;
    if ((rc = st.rc) || (rc = b2_sync_aggregate_verify_dev(ctx, dc, db, dmsg, dsig, n, dok, d48, ctx->s_main))) return rc;
    return st.finish();
}

// ------------------------------------------------------------------------------------------ SkToPk / Sign / hash_to_g2
int b2_sk_to_pk(b2_ctx* ctx, const uint32_t* sk8, uint64_t n, uint8_t* pk48_out) {
    B2_NVTX;
    REQUIRE(ctx && sk8 && pk48_out && n > 0, "sk_to_pk: bad arguments");
    CK(cudaSetDevice(ctx->device));
    staging st(ctx);
    const uint32_t* dsk = st.in(sk8, n * 8);
    uint8_t* dpk = st.out(pk48_out, n * 48);
    if (st.rc) return st.rc;
    k_sk_to_pk<<<blocks_for(n, 64), 64, 0, ctx->s_main>>>(dsk, n, dpk);
    CKL(ctx);
    return st.finish();
}

int b2_hash_to_g2(b2_ctx* ctx, const uint8_t* msg32, uint32_t n_msg, uint8_t* out96) {
    B2_NVTX;
    REQUIRE(ctx && msg32 && out96 && n_msg > 0, "hash_to_g2: bad arguments");
    CK(cudaSetDevice(ctx->device));
    cudaStream_t s = ctx->s_main;
    staging st(ctx);
    const uint8_t* dmsg = st.in(msg32, (size_t)n_msg * 32);
    uint8_t* d96 = st.out(out96, (size_t)n_msg * 96);
    int rc;
    if ((rc = st.rc) || (rc = ensure(ctx, ctx->sc_haff, (size_t)n_msg * 192)) || (rc = ensure(ctx, ctx->sc_hflag, n_msg))) return rc;
    k_hash_to_g2<<<blocks_for(2ull * n_msg, 32), 32, 0, s>>>(dmsg, n_msg, (uint32_t*)ctx->sc_haff.p, (uint8_t*)ctx->sc_hflag.p);
    CKL(ctx);
    k_g2_compress_aff<<<blocks_for(n_msg, 64), 64, 0, s>>>((const uint32_t*)ctx->sc_haff.p, (const uint8_t*)ctx->sc_hflag.p, n_msg, d96);
    CKL(ctx);
    return st.finish();
}

int b2_sign(b2_ctx* ctx, const uint32_t* sk8, const uint32_t* msg_idx, uint64_t n, const uint8_t* msg32, uint32_t n_msg, uint8_t* sig96_out) {
    B2_NVTX;
    REQUIRE(ctx && sk8 && msg_idx && msg32 && sig96_out && n > 0 && n_msg > 0, "sign: bad arguments");
    for (uint64_t i = 0; i < n; i++) REQUIRE(msg_idx[i] < n_msg, "sign: msg_idx out of range");
    CK(cudaSetDevice(ctx->device));
    cudaStream_t s = ctx->s_main;
    staging st(ctx);
    const uint32_t* dsk = st.in(sk8, n * 8);
    const uint32_t* didx = st.in(msg_idx, n);
    const uint8_t* dmsg = st.in(msg32, (size_t)n_msg * 32);
    uint8_t* dsig = st.out(sig96_out, n * 96);
    int rc;
    if ((rc = st.rc) || (rc = ensure(ctx, ctx->sc_haff, (size_t)n_msg * 192)) || (rc = ensure(ctx, ctx->sc_hflag, n_msg))) return rc;
    k_hash_to_g2<<<blocks_for(2ull * n_msg, 32), 32, 0, s>>>(dmsg, n_msg, (uint32_t*)ctx->sc_haff.p, (uint8_t*)ctx->sc_hflag.p);
    CKL(ctx);
    k_sign<<<blocks_for(n, 64), 64, 0, s>>>(dsk, didx, n, (const uint32_t*)ctx->sc_haff.p, dsig);
    CKL(ctx);
    return st.finish();
}

// ------------------------------------------------------------------------------------------ batched SHA-256
int b2_sha256_batch(b2_ctx* ctx, const uint8_t* msgs, uint32_t msg_len, uint64_t n, uint8_t* out32) {
    B2_NVTX;
    REQUIRE(ctx && out32 && n > 0 && (msg_len == 0 || msgs), "sha256_batch: bad arguments");
    CK(cudaSetDevice(ctx->device));
    staging st(ctx);
    const uint8_t* dmsg = st.in(msgs, (size_t)n * msg_len, 16);
    uint8_t* d32 = st.out(out32, (size_t)n * 32);
    if (st.rc) return st.rc;
    k_sha256_fixed<<<blocks_for(n, 128), 128, 0, ctx->s_main>>>(dmsg, msg_len, n, d32);
    CKL(ctx);
    return st.finish();
}

// ------------------------------------------------------------------------------------------ SSZ signing roots
int b2_signing_roots(b2_ctx* ctx, const uint8_t* data128, const uint8_t* domain32, int per_attestation_domain, uint32_t n, uint8_t* out32) {
    B2_NVTX;
    REQUIRE(ctx && data128 && domain32 && out32 && n > 0, "signing_roots: bad arguments");
    CK(cudaSetDevice(ctx->device));
    staging st(ctx);
    const uint8_t* ddata = st.in(data128, (size_t)n * 128);
    const uint8_t* ddom = st.in(domain32, per_attestation_domain ? (size_t)n * 32 : 32);
    uint8_t* d32 = st.out(out32, (size_t)n * 32);
    if (st.rc) return st.rc;
    k_signing_roots<<<blocks_for(n, 64), 64, 0, ctx->s_main>>>(ddata, ddom, per_attestation_domain ? 32u : 0u, n, d32);
    CKL(ctx);
    return st.finish();
}

// ------------------------------------------------------------------------------------------ SSZ wire decode (:714-717)
int b2_attestations_decode(b2_ctx* ctx, const uint8_t* wire, const uint32_t* woff, uint32_t n, uint32_t bits_stride, uint32_t max_bits,
                           uint8_t* bits_out, uint32_t* bit_len_out, uint8_t* data128_out, uint8_t* sig96_out, int32_t* status_out) {
    B2_NVTX;
    REQUIRE(ctx && wire && woff && n > 0 && bits_stride > 0 && bits_out && bit_len_out && data128_out && sig96_out && status_out,
            "attestations_decode: bad arguments");
    int rc;
    if ((rc = check_offsets(ctx, woff, n, "attestations_decode", "woff"))) return rc;
    CK(cudaSetDevice(ctx->device));
    staging st(ctx);
    const uint8_t* dwire = st.in(wire, woff[n], 16);
    const uint32_t* dwoff = st.in(woff, (size_t)n + 1);
    uint8_t* dbits = st.out(bits_out, (size_t)n * bits_stride);
    uint32_t* dlen = st.out(bit_len_out, n);
    uint8_t* ddata = st.out(data128_out, (size_t)n * 128);
    uint8_t* dsig = st.out(sig96_out, (size_t)n * 96);
    int32_t* dst = st.out(status_out, n);
    if (st.rc) return st.rc;
    k_attestations_decode<<<blocks_for((uint64_t)n * 32, 128), 128, 0, ctx->s_main>>>(dwire, dwoff, n, bits_stride, max_bits, dbits, dlen, ddata, dsig, dst);
    CKL(ctx);
    return st.finish();
}

// ------------------------------------------------------------------------------------------ attestation intake (intake.cuh)
// The batch layout both attestation intakes share: one epoch of slots_per_epoch * committees_per_slot committees, an epoch that
// validate_target_epoch_against_current_time accepts for the whole batch (the current slot's epoch or the one before it), and a block
// tree to resolve votes against.  slots_per_epoch > 0.
static int check_intake(b2_ctx* ctx, uint32_t n_committees, uint32_t committees_per_slot, uint32_t slots_per_epoch, uint64_t epoch,
                        uint64_t current_slot, const char* what) {
    if ((uint64_t)committees_per_slot * slots_per_epoch != n_committees)
        return reject(ctx, what, "n_committees must be slots_per_epoch * committees_per_slot");
    const uint64_t cur = current_slot / slots_per_epoch;
    if (current_slot >= (1ull << 63) || !(epoch == cur || (cur > 0 && epoch == cur - 1)))
        return reject(ctx, what, "the epoch must be the current slot's epoch or the one before it");
    if (ctx->n_blocks == 0) return reject(ctx, what, "no tree loaded (b2_tree_load)");
    return B2_OK;
}
static int check_attestation_intake(b2_ctx* ctx, const void* wire, const void* woff, uint32_t n_att, const void* off, uint32_t n_committees,
                                    uint32_t committees_per_slot, uint32_t slots_per_epoch, uint32_t bits_stride, uint64_t epoch, uint64_t current_slot,
                                    const void* domain32, uint32_t max_votes, const void* status_out, const void* vote_out, const void* vote_off_out,
                                    const void* sig96_out, const void* data128_out, const void* msg32_out, const void* source_epoch_out,
                                    const void* target_epoch_out, const void* block_idx_out) {
    REQUIRE(ctx && wire && woff && off && domain32 && status_out && vote_out && vote_off_out && sig96_out && data128_out && msg32_out &&
                source_epoch_out && target_epoch_out && block_idx_out && n_att > 0 && max_votes > 0 && bits_stride > 0 && bits_stride <= 256 &&
                committees_per_slot > 0 && slots_per_epoch > 0,
            "attestation_intake: bad arguments");
    return check_intake(ctx, n_committees, committees_per_slot, slots_per_epoch, epoch, current_slot, "attestation_intake");
}
// Both attestation intakes after their argument checks: d_members == nullptr is the phase 0 form (k_intake_parse), otherwise the
// SingleAttestation form (k_single_parse, which also writes the offset view the later kernels read as woff).
static int attestation_intake_enqueue(b2_ctx* ctx, const uint8_t* d_wire, uint64_t wire_len, const uint32_t* d_woff, uint32_t n_att,
                                      const uint32_t* d_subnet, uint32_t subnet_count, const uint32_t* d_members, const uint32_t* d_off,
                                      uint32_t n_committees, uint64_t n_sig, uint32_t committees_per_slot, uint32_t slots_per_epoch,
                                      uint32_t bits_stride, uint64_t epoch, uint64_t current_slot, const uint8_t* domain32, uint32_t max_votes,
                                      int32_t* d_status_out, uint32_t* d_vote_out, uint32_t* d_vote_off_out, uint8_t* d_sig96_out,
                                      uint8_t* d_data128_out, uint8_t* d_msg32_out, uint64_t* d_source_epoch_out, uint64_t* d_target_epoch_out,
                                      uint32_t* d_block_idx_out, void* stream) {
    REQUIRE(n_sig < (1ull << 32), "attestation_intake: n_sig does not fit 32 bits");      // the host form's n_sig is a u32 offset
    CK(cudaSetDevice(ctx->device));
    const tree_tables& t = ctx->tree;
    intake_args A = {};
    A.wire = d_wire;
    A.wire_len = wire_len;
    A.woff = d_woff;
    A.n_att = n_att;
    A.off = d_off;
    A.n_committees = n_committees;
    A.committees_per_slot = committees_per_slot;
    A.slots_per_epoch = slots_per_epoch;
    A.bits_stride = bits_stride;
    A.n_sig = n_sig;
    A.epoch = epoch;
    A.current_slot = current_slot;
    A.root = t.root;
    A.parent = t.parent;
    A.slot = t.slot;
    A.n_blocks = ctx->n_blocks;
    A.status = d_status_out;
    A.vote = d_vote_out;
    A.vote_off = d_vote_off_out;
    A.sig96 = d_sig96_out;
    A.max_votes = max_votes;
    memcpy(A.domain.b, domain32, 32);
    A.data128 = d_data128_out;
    A.msg32 = d_msg32_out;
    A.source_epoch = d_source_epoch_out;
    A.target_epoch = d_target_epoch_out;
    A.block_idx = d_block_idx_out;
    A.guard = ctx->d_guard;
    const size_t nc = (size_t)n_committees + 1;
    uint32_t* sorted;      // written by k_intake_sorted, read by the kernels through A.sorted
    scratch sc(ctx, ctx->in);
    sc(A.comm, n_att); sc(A.pos, n_att); sc(A.fp, n_att); sc(A.grp, n_att);
    sc(A.bucket, nc); sc(A.cursor, nc); sc(A.nkept, nc);
    sc(A.list, n_att); sc(A.lead, n_att); sc(A.gstat, n_att); sc(A.gblk, n_att); sc(A.gmin, n_att); sc(A.vgrp, n_att);
    sc(A.posatt, n_sig); sc(sorted, ctx->n_blocks);
    single_args S = {};
    if (d_members) sc(S.view, n_att);
    if (sc.rc) return sc.rc;
    A.sorted = sorted;
    cudaStream_t s = (cudaStream_t)stream;
    CK(cudaStreamWaitEvent(s, ctx->ev_intake, 0));
    k_intake_sorted<<<blocks_for(ctx->n_blocks, 256), 256, 0, s>>>(t.rank_id, ctx->n_blocks, sorted);
    CKL(ctx);
    CK(cudaMemsetAsync(A.bucket, 0, nc * 4, s));
    if (d_members) {
        A.woff = S.view;      // the later kernels read each SingleAttestation's data and signature through the offset view
        S.T = A;
        S.woff = d_woff;
        S.members = d_members;
        S.subnet = d_subnet;
        S.subnet_count = subnet_count;
        k_single_parse<<<blocks_for((uint64_t)n_att * 32, 128), 128, 0, s>>>(S);
    } else {
        k_intake_parse<<<blocks_for((uint64_t)n_att * 32, 128), 128, 0, s>>>(A);
    }
    CKL(ctx);
    k_intake_scan<<<1, 1024, 0, s>>>(A.bucket, n_committees, A.cursor);      // bucket[n_committees] = the candidates
    CKL(ctx);
    k_intake_scatter<<<blocks_for(n_att, 256), 256, 0, s>>>(A);
    CKL(ctx);
    k_intake_committee<<<n_committees, INTAKE_THREADS, 0, s>>>(A);
    CKL(ctx);
    k_intake_scan<<<1, 1024, 0, s>>>(d_vote_off_out, n_committees, nullptr);      // vote_off[n_committees] = the epoch's votes
    CKL(ctx);
    k_intake_votes<<<blocks_for(max_votes, 64), 64, 0, s>>>(A);
    CKL(ctx);
    k_intake_sigs<<<n_committees, INTAKE_THREADS, 0, s>>>(A);
    CKL(ctx);
    CK(cudaEventRecord(ctx->ev_intake, s));
    return B2_OK;
}
int b2_attestation_intake_dev(b2_ctx* ctx, const uint8_t* d_wire, uint64_t wire_len, const uint32_t* d_woff, uint32_t n_att, const uint32_t* d_off,
                              uint32_t n_committees, uint64_t n_sig, uint32_t committees_per_slot, uint32_t slots_per_epoch, uint32_t bits_stride,
                              uint64_t epoch, uint64_t current_slot, const uint8_t* domain32, uint32_t max_votes, int32_t* d_status_out,
                              uint32_t* d_vote_out, uint32_t* d_vote_off_out, uint8_t* d_sig96_out, uint8_t* d_data128_out, uint8_t* d_msg32_out,
                              uint64_t* d_source_epoch_out, uint64_t* d_target_epoch_out, uint32_t* d_block_idx_out, void* stream) {
    B2_NVTX;
    int rc;
    if ((rc = check_attestation_intake(ctx, d_wire, d_woff, n_att, d_off, n_committees, committees_per_slot, slots_per_epoch, bits_stride, epoch, current_slot, domain32,
                                       max_votes, d_status_out, d_vote_out, d_vote_off_out, d_sig96_out, d_data128_out, d_msg32_out, d_source_epoch_out,
                                       d_target_epoch_out, d_block_idx_out)))
        return rc;
    return attestation_intake_enqueue(ctx, d_wire, wire_len, d_woff, n_att, nullptr, 0, nullptr, d_off, n_committees, n_sig, committees_per_slot,
                                      slots_per_epoch, bits_stride, epoch, current_slot, domain32, max_votes, d_status_out, d_vote_out, d_vote_off_out,
                                      d_sig96_out, d_data128_out, d_msg32_out, d_source_epoch_out, d_target_epoch_out, d_block_idx_out, stream);
}
// the SingleAttestation form's arguments: the phase 0 form's, the members and the arrival subnets
static int check_single_attestation_intake(b2_ctx* ctx, const void* wire, const void* woff, uint32_t n_att, const void* subnet, uint32_t subnet_count,
                                           const void* members, const void* off, uint32_t n_committees, uint32_t committees_per_slot,
                                           uint32_t slots_per_epoch, uint32_t bits_stride, uint64_t epoch, uint64_t current_slot, const void* domain32,
                                           uint32_t max_votes, const void* status_out, const void* vote_out, const void* vote_off_out,
                                           const void* sig96_out, const void* data128_out, const void* msg32_out, const void* source_epoch_out,
                                           const void* target_epoch_out, const void* block_idx_out) {
    REQUIRE(ctx && subnet && members && subnet_count > 0, "single_attestation_intake: bad arguments");
    return check_attestation_intake(ctx, wire, woff, n_att, off, n_committees, committees_per_slot, slots_per_epoch, bits_stride, epoch, current_slot,
                                    domain32, max_votes, status_out, vote_out, vote_off_out, sig96_out, data128_out, msg32_out, source_epoch_out,
                                    target_epoch_out, block_idx_out);
}
int b2_single_attestation_intake_dev(b2_ctx* ctx, const uint8_t* d_wire, uint64_t wire_len, const uint32_t* d_woff, uint32_t n_att,
                                     const uint32_t* d_subnet, uint32_t subnet_count, const uint32_t* d_members, const uint32_t* d_off,
                                     uint32_t n_committees, uint64_t n_sig, uint32_t committees_per_slot, uint32_t slots_per_epoch, uint32_t bits_stride,
                                     uint64_t epoch, uint64_t current_slot, const uint8_t* domain32, uint32_t max_votes, int32_t* d_status_out,
                                     uint32_t* d_vote_out, uint32_t* d_vote_off_out, uint8_t* d_sig96_out, uint8_t* d_data128_out, uint8_t* d_msg32_out,
                                     uint64_t* d_source_epoch_out, uint64_t* d_target_epoch_out, uint32_t* d_block_idx_out, void* stream) {
    B2_NVTX;
    int rc;
    if ((rc = check_single_attestation_intake(ctx, d_wire, d_woff, n_att, d_subnet, subnet_count, d_members, d_off, n_committees, committees_per_slot,
                                              slots_per_epoch, bits_stride, epoch, current_slot, domain32, max_votes, d_status_out, d_vote_out,
                                              d_vote_off_out, d_sig96_out, d_data128_out, d_msg32_out, d_source_epoch_out, d_target_epoch_out,
                                              d_block_idx_out)))
        return rc;
    return attestation_intake_enqueue(ctx, d_wire, wire_len, d_woff, n_att, d_subnet, subnet_count, d_members, d_off, n_committees, n_sig,
                                      committees_per_slot, slots_per_epoch, bits_stride, epoch, current_slot, domain32, max_votes, d_status_out,
                                      d_vote_out, d_vote_off_out, d_sig96_out, d_data128_out, d_msg32_out, d_source_epoch_out, d_target_epoch_out,
                                      d_block_idx_out, stream);
}

// Both host forms after their argument checks: stage, zero the vote rows, enqueue (members == nullptr: the phase 0 form).
static int attestation_intake_host(b2_ctx* ctx, const uint8_t* wire, uint64_t wire_len, const uint32_t* woff, uint32_t n_att, const uint32_t* subnet,
                                   uint32_t subnet_count, const uint32_t* members, const uint32_t* off, uint32_t n_committees,
                                   uint32_t committees_per_slot, uint32_t slots_per_epoch, uint32_t bits_stride, uint64_t epoch, uint64_t current_slot,
                                   const uint8_t* domain32, uint32_t max_votes, int32_t* status_out, uint32_t* vote_out, uint32_t* vote_off_out,
                                   uint8_t* sig96_out, uint8_t* data128_out, uint8_t* msg32_out, uint64_t* source_epoch_out, uint64_t* target_epoch_out,
                                   uint32_t* block_idx_out) {
    int rc;
    if ((rc = check_wire(ctx, woff, n_att, wire_len, "attestation_intake")) ||
        (rc = check_committees(ctx, off, n_committees, bits_stride, "attestation_intake")))
        return rc;
    const uint64_t n_sig = off[n_committees];
    CK(cudaSetDevice(ctx->device));
    staging st(ctx);
    const uint8_t* dwire = st.in(wire, wire_len, 16);
    const uint32_t* dwoff = st.in(woff, (size_t)n_att + 1);
    const uint32_t* dsub = members ? st.in(subnet, n_att) : nullptr;
    const uint32_t* dmem = members ? st.in(members, n_sig, 4) : nullptr;
    const uint32_t* doff = st.in(off, (size_t)n_committees + 1);
    int32_t* dst = st.out(status_out, n_att);
    uint32_t* dvote = st.out(vote_out, n_sig);
    uint32_t* dvoff = st.out(vote_off_out, (size_t)n_committees + 1);
    uint8_t* dsig = st.out(sig96_out, n_sig * 96);
    uint8_t* ddata = st.out(data128_out, (size_t)max_votes * 128);
    uint8_t* dmsg = st.out(msg32_out, (size_t)max_votes * 32);
    uint64_t* dsrc = st.out(source_epoch_out, max_votes);
    uint64_t* dtgt = st.out(target_epoch_out, max_votes);
    uint32_t* dblk = st.out(block_idx_out, max_votes);
    if (st.rc) return st.rc;
    // rows past the epoch's vote count are zero
    CK(cudaMemsetAsync(ddata, 0, (size_t)max_votes * 128, ctx->s_main));
    CK(cudaMemsetAsync(dmsg, 0, (size_t)max_votes * 32, ctx->s_main));
    CK(cudaMemsetAsync(dsrc, 0, (size_t)max_votes * 8, ctx->s_main));
    CK(cudaMemsetAsync(dtgt, 0, (size_t)max_votes * 8, ctx->s_main));
    CK(cudaMemsetAsync(dblk, 0, (size_t)max_votes * 4, ctx->s_main));
    if ((rc = attestation_intake_enqueue(ctx, dwire, wire_len, dwoff, n_att, dsub, subnet_count, dmem, doff, n_committees, n_sig, committees_per_slot,
                                         slots_per_epoch, bits_stride, epoch, current_slot, domain32, max_votes, dst, dvote, dvoff, dsig, ddata, dmsg,
                                         dsrc, dtgt, dblk, ctx->s_main)))
        return rc;
    return st.finish();
}
int b2_attestation_intake(b2_ctx* ctx, const uint8_t* wire, uint64_t wire_len, const uint32_t* woff, uint32_t n_att, const uint32_t* off,
                          uint32_t n_committees, uint32_t committees_per_slot, uint32_t slots_per_epoch, uint32_t bits_stride, uint64_t epoch,
                          uint64_t current_slot, const uint8_t* domain32, uint32_t max_votes, int32_t* status_out, uint32_t* vote_out,
                          uint32_t* vote_off_out, uint8_t* sig96_out, uint8_t* data128_out, uint8_t* msg32_out, uint64_t* source_epoch_out,
                          uint64_t* target_epoch_out, uint32_t* block_idx_out) {
    B2_NVTX;
    if (int rc = check_attestation_intake(ctx, wire, woff, n_att, off, n_committees, committees_per_slot, slots_per_epoch, bits_stride, epoch, current_slot,
                                          domain32, max_votes, status_out, vote_out, vote_off_out, sig96_out, data128_out, msg32_out, source_epoch_out,
                                          target_epoch_out, block_idx_out))
        return rc;
    return attestation_intake_host(ctx, wire, wire_len, woff, n_att, nullptr, 0, nullptr, off, n_committees, committees_per_slot, slots_per_epoch,
                                   bits_stride, epoch, current_slot, domain32, max_votes, status_out, vote_out, vote_off_out, sig96_out, data128_out,
                                   msg32_out, source_epoch_out, target_epoch_out, block_idx_out);
}
int b2_single_attestation_intake(b2_ctx* ctx, const uint8_t* wire, uint64_t wire_len, const uint32_t* woff, uint32_t n_att, const uint32_t* subnet,
                                 uint32_t subnet_count, const uint32_t* members, const uint32_t* off, uint32_t n_committees, uint32_t committees_per_slot,
                                 uint32_t slots_per_epoch, uint32_t bits_stride, uint64_t epoch, uint64_t current_slot, const uint8_t* domain32,
                                 uint32_t max_votes, int32_t* status_out, uint32_t* vote_out, uint32_t* vote_off_out, uint8_t* sig96_out,
                                 uint8_t* data128_out, uint8_t* msg32_out, uint64_t* source_epoch_out, uint64_t* target_epoch_out,
                                 uint32_t* block_idx_out) {
    B2_NVTX;
    if (int rc = check_single_attestation_intake(ctx, wire, woff, n_att, subnet, subnet_count, members, off, n_committees, committees_per_slot,
                                                 slots_per_epoch, bits_stride, epoch, current_slot, domain32, max_votes, status_out, vote_out,
                                                 vote_off_out, sig96_out, data128_out, msg32_out, source_epoch_out, target_epoch_out, block_idx_out))
        return rc;
    return attestation_intake_host(ctx, wire, wire_len, woff, n_att, subnet, subnet_count, members, off, n_committees, committees_per_slot,
                                   slots_per_epoch, bits_stride, epoch, current_slot, domain32, max_votes, status_out, vote_out, vote_off_out,
                                   sig96_out, data128_out, msg32_out, source_epoch_out, target_epoch_out, block_idx_out);
}

// ------------------------------------------------------------------------------------------ aggregated-attestation intake (aggintake.cuh)
static int check_aggregate_and_proof_intake(b2_ctx* ctx, const void* wire, const void* woff, uint32_t n, const void* members, const void* off,
                                            uint32_t n_committees, uint32_t committees_per_slot, uint32_t slots_per_epoch, uint32_t bits_stride,
                                            uint64_t epoch, uint64_t current_slot, const void* domains96, uint32_t target_aggregators, const void* status_out,
                                            const void* committee_out, const void* data_id_out, const void* bits_out, const void* sig96_out,
                                            const void* msg32_out, const void* target_epoch_out, const void* block_idx_out, const void* members_out,
                                            const void* item_off_out) {
    REQUIRE(ctx && wire && woff && members && off && domains96 && status_out && committee_out && data_id_out && bits_out && sig96_out && msg32_out &&
                target_epoch_out && block_idx_out && members_out && item_off_out && n > 0 && n < (1u << 28) && bits_stride > 0 && bits_stride <= 256 &&
                (uint64_t)n * 8 * bits_stride < (1ull << 32) && committees_per_slot > 0 && slots_per_epoch > 0 && target_aggregators > 0,
            "aggregate_and_proof_intake: bad arguments");
    if (int rc = check_intake(ctx, n_committees, committees_per_slot, slots_per_epoch, epoch, current_slot, "aggregate_and_proof_intake")) return rc;
    return ctx->n_val > 0 ? B2_OK : reject(ctx, "aggregate_and_proof_intake", "registry not loaded");
}
int b2_aggregate_and_proof_intake_dev(b2_ctx* ctx, const uint8_t* d_wire, uint64_t wire_len, const uint32_t* d_woff, uint32_t n, const uint32_t* d_members,
                                      const uint32_t* d_off, uint32_t n_committees, uint64_t n_sig, uint32_t committees_per_slot, uint32_t slots_per_epoch,
                                      uint32_t bits_stride, uint64_t epoch, uint64_t current_slot, const uint8_t* domains96, uint32_t target_aggregators,
                                      uint64_t propagation_slot_range, int32_t* d_status_out, uint32_t* d_committee_out, uint32_t* d_data_id_out,
                                      uint8_t* d_bits_out, uint8_t* d_sig96_out, uint8_t* d_msg32_out, uint64_t* d_target_epoch_out,
                                      uint32_t* d_block_idx_out, uint32_t* d_members_out, uint32_t* d_item_off_out, void* stream) {
    B2_NVTX;
    int rc;
    if ((rc = check_aggregate_and_proof_intake(ctx, d_wire, d_woff, n, d_members, d_off, n_committees, committees_per_slot, slots_per_epoch, bits_stride, epoch,
                                               current_slot, domains96, target_aggregators, d_status_out, d_committee_out, d_data_id_out, d_bits_out,
                                               d_sig96_out, d_msg32_out, d_target_epoch_out, d_block_idx_out, d_members_out, d_item_off_out)))
        return rc;
    REQUIRE(n_sig < (1ull << 32), "aggregate_and_proof_intake: n_sig does not fit 32 bits");      // the host form's n_sig is a u32 offset
    CK(cudaSetDevice(ctx->device));
    uint32_t tab = 1;
    while (tab < 2 * n) tab <<= 1;
    const tree_tables& t = ctx->tree;
    api_args A = {};
    intake_args& T = A.T;
    T.n_att = n;
    T.off = d_off;
    T.n_committees = n_committees;
    T.committees_per_slot = committees_per_slot;
    T.slots_per_epoch = slots_per_epoch;
    T.bits_stride = bits_stride;
    T.n_sig = n_sig;
    T.epoch = epoch;
    T.current_slot = current_slot;
    T.root = t.root;
    T.parent = t.parent;
    T.slot = t.slot;
    T.n_blocks = ctx->n_blocks;
    T.guard = ctx->d_guard;
    A.wire = d_wire;
    A.wire_len = wire_len;
    A.woff = d_woff;
    A.n = n;
    A.members = d_members;
    A.committees_per_slot = committees_per_slot;
    A.slots_per_epoch = slots_per_epoch;
    A.bits_stride = bits_stride;
    A.target_aggregators = target_aggregators;
    A.epoch = epoch;
    A.current_slot = current_slot;
    A.propagation_range = propagation_slot_range;
    A.n_val = ctx->n_val;
    A.dtab_mask = tab - 1;
    A.status = d_status_out;
    A.committee = d_committee_out;
    A.data_id = d_data_id_out;
    A.bits = d_bits_out;
    A.sig96 = d_sig96_out;
    A.msg32 = d_msg32_out;
    A.target_epoch = d_target_epoch_out;
    A.block_idx = d_block_idx_out;
    A.members_out = d_members_out;
    A.item_off = d_item_off_out;
    memcpy(A.dom_att.b, domains96, 32);
    memcpy(A.dom_sel.b, domains96 + 32, 32);
    memcpy(A.dom_aap.b, domains96 + 64, 32);
    A.guard = ctx->d_guard;
    const size_t nc = (size_t)n_committees + 1;
    uint8_t *fav_ok, *av_ok;      // written by the verify helpers, read by the kernels through A
    uint32_t* sorted;             // written by k_intake_sorted, read through T.sorted
    scratch sc(ctx, ctx->api);
    sc(T.comm, n); sc(A.fp, n); sc(A.slot_of, n); sc(A.dtab, tab); sc(A.dmin, tab); sc(T.list, n); sc(A.acc, n); sc(A.accepted_by, ctx->n_val);
    sc(A.incomm, n); sc(A.tst, n); sc(A.fbits, (size_t)n * bits_stride, 16); sc(fav_ok, n);
    sc(T.bucket, nc); sc(T.cursor, nc); sc(sorted, ctx->n_blocks);
    sc(A.av_signer, 2 * (size_t)n); sc(A.av_off, 2 * (size_t)n + 1); sc(A.av_msg, (size_t)n * 64); sc(A.av_sig, (size_t)n * 192); sc(av_ok, 2 * (size_t)n);
    if (sc.rc) return sc.rc;
    A.fav_ok = fav_ok;
    A.av_ok = av_ok;
    T.sorted = sorted;
    cudaStream_t s = (cudaStream_t)stream;
    CK(cudaStreamWaitEvent(s, ctx->ev_intake, 0));
    k_intake_sorted<<<blocks_for(ctx->n_blocks, 256), 256, 0, s>>>(t.rank_id, ctx->n_blocks, sorted);
    CKL(ctx);
    CK(cudaMemsetAsync(T.bucket, 0, nc * 4, s));
    CK(cudaMemsetAsync(A.dtab, 0xff, (size_t)tab * 4, s));
    CK(cudaMemsetAsync(A.dmin, 0xff, (size_t)tab * 4, s));
    CK(cudaMemsetAsync(A.accepted_by, 0xff, ctx->n_val * 4, s));
    k_api_parse<<<blocks_for((uint64_t)n * 32, 128), 128, 0, s>>>(A);
    CKL(ctx);
    k_api_data<<<blocks_for(n, 128), 128, 0, s>>>(A);
    CKL(ctx);
    k_api_roots<<<blocks_for(n, 64), 64, 0, s>>>(A);
    CKL(ctx);
    k_api_sets<<<blocks_for(n, 64), 64, 0, s>>>(A);
    CKL(ctx);
    // FastAggregateVerify of the aggregates over their member rows, then AggregateVerify of the 2n single-key sets
    pk_source P = {d_members_out, d_item_off_out, A.fbits, bits_stride, nullptr, 0};
    if ((rc = verify_fork(ctx, ctx->slot[0], P, d_msg32_out, n, s)) || (rc = verify_main(ctx, ctx->slot[0], d_sig96_out, n, fav_ok, s))) return rc;
    if ((rc = aggregate_verify_enqueue(ctx, A.av_signer, nullptr, A.av_msg, A.av_off, 2ull * n, A.av_sig, 2 * n, av_ok, s))) return rc;
    k_intake_scan<<<1, 1024, 0, s>>>(T.bucket, n_committees, T.cursor);      // bucket[n_committees] = the candidates
    CKL(ctx);
    k_intake_scatter<<<blocks_for(n, 256), 256, 0, s>>>(T);
    CKL(ctx);
    k_api_committee<<<n_committees, 32, 0, s>>>(A);
    CKL(ctx);
    k_api_outsiders<<<blocks_for(n, 128), 128, 0, s>>>(A);
    CKL(ctx);
    CK(cudaEventRecord(ctx->ev_intake, s));
    return B2_OK;
}

int b2_aggregate_and_proof_intake(b2_ctx* ctx, const uint8_t* wire, uint64_t wire_len, const uint32_t* woff, uint32_t n, const uint32_t* members,
                                  const uint32_t* off, uint32_t n_committees, uint32_t committees_per_slot, uint32_t slots_per_epoch, uint32_t bits_stride,
                                  uint64_t epoch, uint64_t current_slot, const uint8_t* domains96, uint32_t target_aggregators,
                                  uint64_t propagation_slot_range, int32_t* status_out, uint32_t* committee_out, uint32_t* data_id_out, uint8_t* bits_out,
                                  uint8_t* sig96_out, uint8_t* msg32_out, uint64_t* target_epoch_out, uint32_t* block_idx_out, uint32_t* members_out,
                                  uint32_t* item_off_out) {
    B2_NVTX;
    int rc;
    if ((rc = check_aggregate_and_proof_intake(ctx, wire, woff, n, members, off, n_committees, committees_per_slot, slots_per_epoch, bits_stride, epoch, current_slot,
                                               domains96, target_aggregators, status_out, committee_out, data_id_out, bits_out, sig96_out, msg32_out,
                                               target_epoch_out, block_idx_out, members_out, item_off_out)) ||
        (rc = check_wire(ctx, woff, n, wire_len, "aggregate_and_proof_intake")) ||
        (rc = check_committees(ctx, off, n_committees, bits_stride, "aggregate_and_proof_intake")))
        return rc;
    const uint64_t n_sig = off[n_committees], W = 8ull * bits_stride;
    CK(cudaSetDevice(ctx->device));
    staging st(ctx);
    const uint8_t* dwire = st.in(wire, wire_len, 16);
    const uint32_t* dwoff = st.in(woff, (size_t)n + 1);
    const uint32_t* dmem = st.in(members, n_sig, 4);
    const uint32_t* doff = st.in(off, (size_t)n_committees + 1);
    int32_t* dst = st.out(status_out, n);
    uint32_t* dcom = st.out(committee_out, n);
    uint32_t* ddid = st.out(data_id_out, n);
    uint8_t* dbits = st.out(bits_out, (size_t)n * bits_stride);
    uint8_t* dsig = st.out(sig96_out, (size_t)n * 96);
    uint8_t* dmsg = st.out(msg32_out, (size_t)n * 32);
    uint64_t* dtgt = st.out(target_epoch_out, n);
    uint32_t* dblk = st.out(block_idx_out, n);
    uint32_t* dmo = st.out(members_out, n * W);
    uint32_t* dio = st.out(item_off_out, (size_t)n + 1);
    if (st.rc) return st.rc;
    if ((rc = b2_aggregate_and_proof_intake_dev(ctx, dwire, wire_len, dwoff, n, dmem, doff, n_committees, n_sig, committees_per_slot, slots_per_epoch,
                                                bits_stride, epoch, current_slot, domains96, target_aggregators, propagation_slot_range, dst, dcom, ddid,
                                                dbits, dsig, dmsg, dtgt, dblk, dmo, dio, ctx->s_main)))
        return rc;
    return st.finish();
}

// ------------------------------------------------------------------------------------------ block attestations (blockatt.cuh, blockatt_electra.cuh)
// The phase 0 call (b2_block_attestations) and the Electra call (b2_block_attestations_electra) differ only in the decode and checks
// 1-12 of each attestation (k_ba_parse, or k_bae_parse and k_bae_rows) and in the member rows those write; the argument checks, the
// signature check, block atomicity, the flag scatter and the proposer rewards are one sequence for both.
static uint32_t isqrt_u32(uint32_t n) {
    uint32_t x = 0;
    while ((uint64_t)(x + 1) * (x + 1) <= n) x++;
    return x;
}
// R: the Electra member rows' padded length, a whole number of split-sum chunks
static uint64_t bae_row(uint32_t row_max) { return (uint64_t)BAE_CHUNK * (((uint64_t)row_max + BAE_CHUNK - 1) / BAE_CHUNK); }

// A call's form and member-row shape.  Phase 0: bits_stride, the committees' bit-row stride.  Electra: M committees per slot of at most
// max_vpc members each, and row_max, the largest member count of one slot's committees (the host form derives it from off).
struct ba_form {
    bool electra;
    uint32_t bits_stride, M, max_vpc, row_max;
    const char* what() const { return electra ? "block_attestations_electra" : "block_attestations"; }
    uint64_t width() const { return electra ? bae_row(row_max) : 8ull * bits_stride; }      // members per attestation row
};

// what both calls take alike: everything but the member-row shape
static int check_block_attestations(b2_ctx* ctx, const char* what, const void* wire, const void* woff, uint32_t n_att, const void* block_off,
                                    const void* block_slot, uint32_t n_blocks, const void* members, const void* off, uint32_t n_committees,
                                    uint32_t cps_prev, uint32_t cps_cur, const void* chain_roots, const void* justified80, const void* domains64,
                                    uint32_t slots_per_epoch, uint32_t min_inclusion_delay, uint64_t effective_balance_increment, const void* status_out,
                                    const void* flag_mask_out, const void* numerator_out, const void* block_status_out, const void* block_first_out,
                                    const void* block_reward_out, const void* n_applied_out) {
    if (!ctx) return B2_EINVAL;
    if (!(wire && woff && block_off && block_slot && members && off && chain_roots && justified80 && domains64 && status_out && flag_mask_out &&
          numerator_out && block_status_out && block_first_out && block_reward_out && n_applied_out && n_att > 0 && n_att < (1u << 28) &&
          n_blocks > 0 && slots_per_epoch > 0 && cps_cur > 0 && ((uint64_t)cps_prev + cps_cur) * slots_per_epoch < (1ull << 31) &&
          min_inclusion_delay > 0 && effective_balance_increment > 0))
        return reject(ctx, what, "bad arguments");
    if (((uint64_t)cps_prev + cps_cur) * slots_per_epoch != n_committees)
        return reject(ctx, what, "n_committees must be slots_per_epoch * (cps_prev + cps_cur)");
    if (ctx->n_val == 0) return reject(ctx, what, "registry not loaded");
    return ctx->reg.part[0] && ctx->reg.part[1] ? B2_OK : reject(ctx, what, "both participation tables must be loaded (b2_participation_load)");
}
// the form's member-row shape; every row of the call fits u32 member offsets
static int check_ba_shape(b2_ctx* ctx, uint32_t n_att, const ba_form& f) {
    const bool ok = f.electra ? f.M >= 1 && f.M <= 64 && f.max_vpc > 0 && (uint64_t)f.max_vpc * f.M < (1ull << 31) && f.row_max > 0
                              : f.bits_stride > 0 && f.bits_stride <= 256;
    return ok && n_att * f.width() < (1ull << 32) ? B2_OK : reject(ctx, f.what(), "bad arguments");
}

// Both calls after their argument checks; only the parse step depends on the form.
static int block_attestations_enqueue(b2_ctx* ctx, const ba_form& f, const uint8_t* d_wire, uint64_t wire_len, const uint32_t* d_woff, uint32_t n_att,
                                      const uint32_t* d_block_off, const uint64_t* d_block_slot, uint32_t n_blocks, const uint32_t* d_members,
                                      const uint32_t* d_off, uint64_t n_sig, uint32_t cps_prev, uint32_t cps_cur, const uint8_t* d_chain_roots,
                                      const uint8_t* justified80, const uint8_t* domains64, uint32_t slots_per_epoch, uint32_t min_inclusion_delay,
                                      uint64_t effective_balance_increment, uint64_t base_reward_per_increment, int32_t* d_status_out,
                                      uint8_t* d_flag_mask_out, uint64_t* d_numerator_out, int32_t* d_block_status_out, uint32_t* d_block_first_out,
                                      uint64_t* d_block_reward_out, uint32_t* d_n_applied_out, void* stream) {
    if (n_sig >= (1ull << 32)) return reject(ctx, f.what(), "n_sig does not fit 32 bits");      // the host form's n_sig is a u32 offset
    CK(cudaSetDevice(ctx->device));
    const size_t n = n_att, W = f.width();
    bae_args E = {};      // the Electra kernels' arguments; the phase 0 ones are E.B
    ba_args& A = E.B;
    A.wire = d_wire;
    A.wire_len = wire_len;
    A.woff = d_woff;
    A.n = n_att;
    A.block_off = d_block_off;
    A.block_slot = d_block_slot;
    A.n_blocks = n_blocks;
    A.members = d_members;
    A.T.off = d_off;
    A.T.n_sig = n_sig;
    A.T.bits_stride = (uint32_t)(W / 8);
    A.cps_prev = cps_prev;
    A.cps_cur = cps_cur;
    A.slots_per_epoch = slots_per_epoch;
    A.bits_stride = (uint32_t)(W / 8);
    A.min_delay = min_inclusion_delay;
    A.isqrt_spe = isqrt_u32(slots_per_epoch);
    A.chain_roots = d_chain_roots;
    memcpy(A.justified.b, justified80, 80);
    memcpy(A.dom[0].b, domains64, 32);
    memcpy(A.dom[1].b, domains64 + 32, 32);
    A.status = d_status_out;
    A.flag_mask = d_flag_mask_out;
    A.numerator = (unsigned long long*)d_numerator_out;
    A.block_status = d_block_status_out;
    A.block_first = d_block_first_out;
    A.block_reward = (unsigned long long*)d_block_reward_out;
    A.n_applied = d_n_applied_out;
    A.guard = ctx->d_guard;
    uint8_t* msg32;
    scratch sc(ctx, ctx->ba);
    sc(A.blk_of, n); sc(A.cur, n); sc(A.fav_ok, n); sc(A.accept, 2 * n); sc(A.num1, n); sc(A.bits, n * W / 8, 16);
    sc(A.sig96, n * 96); sc(A.data128, n * 128); sc(A.dom32, n * 32); sc(msg32, n * 32); sc(A.members_out, n * W); sc(A.item_off, n + 1);
    // FastAggregateVerify's keys: each member row, or in the Electra form the split sum over its BAE_CHUNK-member chunks
    pk_source P = {A.members_out, A.item_off, A.bits, A.bits_stride, nullptr, 0};
    if (f.electra) {
        E.M = f.M;
        E.max_vpc = f.max_vpc;
        E.row_max = f.row_max;
        E.R = (uint32_t)W;
        E.n_chunks = (uint32_t)(W / BAE_CHUNK);
        E.n_sig = n_sig;
        E.off = d_off;
        uint8_t* part_st;
        uint32_t* part_jac;
        sc(E.nbits, n); sc(E.c0, n); sc(E.cmask, n); sc(E.chunk_off, n * E.n_chunks + 1); sc(part_jac, n * E.n_chunks * 36); sc(part_st, n * E.n_chunks);
        P = {A.members_out, E.chunk_off, A.bits, BAE_CHUNK / 8, nullptr, 0, nullptr, nullptr, E.n_chunks, part_jac, part_st};
    }
    if (sc.rc) return sc.rc;
    cudaStream_t s = (cudaStream_t)stream;
    if (f.electra) {
        k_bae_parse<<<blocks_for((uint64_t)n_att * 32, 128), 128, 0, s>>>(E);
        CKL(ctx);
        k_bae_rows<<<n_att, 256, 0, s>>>(E);
    } else {
        k_ba_parse<<<blocks_for((uint64_t)n_att * 32, 128), 128, 0, s>>>(A);
    }
    CKL(ctx);
    k_signing_roots<<<blocks_for(n_att, 64), 64, 0, s>>>(A.data128, A.dom32, 32u, n_att, msg32);
    CKL(ctx);
    int rc;
    if ((rc = verify_fork(ctx, ctx->slot[0], P, msg32, n_att, s)) || (rc = verify_main(ctx, ctx->slot[0], A.sig96, n_att, A.fav_ok, s))) return rc;
    k_ba_blocks<<<1, BA_BLOCKS_THREADS, 0, s>>>(A, f.electra ? 13 : 11);      // the status of a failed FastAggregateVerify
    CKL(ctx);
    // the flag scatter of :745-749, order-exact over (block, list) order: table 0 (target e) writes `numerator`, table 1 (target e - 1) num1
    const registry_tables& R = ctx->reg;
    for (int which = 0; which < 2; which++) {
        const uint8_t* acc = A.accept + (size_t)which * n;
        unsigned long long* num = which == 0 ? A.numerator : A.num1;
        k_part_phase1<<<n_att, 128, 0, s>>>(A.members_out, A.item_off, A.bits, A.bits_stride, d_flag_mask_out, acc, n_att, R.part[which], R.part_first);
        CKL(ctx);
        k_part_phase2<<<n_att, 128, 0, s>>>(A.members_out, A.item_off, A.bits, A.bits_stride, d_flag_mask_out, acc, n_att, R.part_first, R.eff,
                                            effective_balance_increment, base_reward_per_increment, num);
        CKL(ctx);
        k_part_phase3<<<n_att, 128, 0, s>>>(A.members_out, A.item_off, A.bits, A.bits_stride, d_flag_mask_out, acc, n_att, R.part_first, R.part[which]);
        CKL(ctx);
    }
    k_ba_rewards<<<blocks_for((uint64_t)n_blocks * 32, 128), 128, 0, s>>>(A);
    CKL(ctx);
    return B2_OK;
}
int b2_block_attestations_dev(b2_ctx* ctx, const uint8_t* d_wire, uint64_t wire_len, const uint32_t* d_woff, uint32_t n_att, const uint32_t* d_block_off,
                              const uint64_t* d_block_slot, uint32_t n_blocks, const uint32_t* d_members, const uint32_t* d_off, uint32_t n_committees,
                              uint64_t n_sig,
                              uint32_t cps_prev, uint32_t cps_cur, const uint8_t* d_chain_roots, const uint8_t* justified80, const uint8_t* domains64,
                              uint32_t slots_per_epoch, uint32_t min_inclusion_delay, uint32_t bits_stride, uint64_t effective_balance_increment,
                              uint64_t base_reward_per_increment, int32_t* d_status_out, uint8_t* d_flag_mask_out, uint64_t* d_numerator_out,
                              int32_t* d_block_status_out, uint32_t* d_block_first_out, uint64_t* d_block_reward_out, uint32_t* d_n_applied_out,
                              void* stream) {
    B2_NVTX;
    const ba_form f = {false, bits_stride, 0, 0, 0};
    int rc;
    if ((rc = check_block_attestations(ctx, f.what(), d_wire, d_woff, n_att, d_block_off, d_block_slot, n_blocks, d_members, d_off, n_committees, cps_prev,
                                       cps_cur, d_chain_roots, justified80, domains64, slots_per_epoch, min_inclusion_delay, effective_balance_increment,
                                       d_status_out, d_flag_mask_out, d_numerator_out, d_block_status_out, d_block_first_out, d_block_reward_out,
                                       d_n_applied_out)) ||
        (rc = check_ba_shape(ctx, n_att, f)))
        return rc;
    return block_attestations_enqueue(ctx, f, d_wire, wire_len, d_woff, n_att, d_block_off, d_block_slot, n_blocks, d_members, d_off, n_sig, cps_prev,
                                      cps_cur, d_chain_roots, justified80, domains64, slots_per_epoch, min_inclusion_delay, effective_balance_increment,
                                      base_reward_per_increment, d_status_out, d_flag_mask_out, d_numerator_out, d_block_status_out, d_block_first_out,
                                      d_block_reward_out, d_n_applied_out, stream);
}
int b2_block_attestations_electra_dev(b2_ctx* ctx, const uint8_t* d_wire, uint64_t wire_len, const uint32_t* d_woff, uint32_t n_att,
                                      const uint32_t* d_block_off, const uint64_t* d_block_slot, uint32_t n_blocks, const uint32_t* d_members,
                                      const uint32_t* d_off, uint32_t n_committees, uint64_t n_sig, uint32_t cps_prev, uint32_t cps_cur,
                                      const uint8_t* d_chain_roots, const uint8_t* justified80, const uint8_t* domains64, uint32_t slots_per_epoch,
                                      uint32_t min_inclusion_delay, uint32_t max_committees_per_slot, uint32_t max_validators_per_committee,
                                      uint32_t row_max, uint64_t effective_balance_increment, uint64_t base_reward_per_increment,
                                      int32_t* d_status_out, uint8_t* d_flag_mask_out, uint64_t* d_numerator_out, int32_t* d_block_status_out,
                                      uint32_t* d_block_first_out, uint64_t* d_block_reward_out, uint32_t* d_n_applied_out, void* stream) {
    B2_NVTX;
    const ba_form f = {true, 0, max_committees_per_slot, max_validators_per_committee, row_max};
    int rc;
    if ((rc = check_block_attestations(ctx, f.what(), d_wire, d_woff, n_att, d_block_off, d_block_slot, n_blocks, d_members, d_off, n_committees, cps_prev,
                                       cps_cur, d_chain_roots, justified80, domains64, slots_per_epoch, min_inclusion_delay, effective_balance_increment,
                                       d_status_out, d_flag_mask_out, d_numerator_out, d_block_status_out, d_block_first_out, d_block_reward_out,
                                       d_n_applied_out)) ||
        (rc = check_ba_shape(ctx, n_att, f)))
        return rc;
    return block_attestations_enqueue(ctx, f, d_wire, wire_len, d_woff, n_att, d_block_off, d_block_slot, n_blocks, d_members, d_off, n_sig, cps_prev,
                                      cps_cur, d_chain_roots, justified80, domains64, slots_per_epoch, min_inclusion_delay, effective_balance_increment,
                                      base_reward_per_increment, d_status_out, d_flag_mask_out, d_numerator_out, d_block_status_out, d_block_first_out,
                                      d_block_reward_out, d_n_applied_out, stream);
}

// Both host forms: the argument checks, the checks that read the host arrays (the Electra form derives row_max here), stage, enqueue.
static int block_attestations_host(b2_ctx* ctx, ba_form f, const uint8_t* wire, uint64_t wire_len, const uint32_t* woff, uint32_t n_att,
                                   const uint32_t* block_off, const uint64_t* block_slot, uint32_t n_blocks, const uint32_t* members, const uint32_t* off,
                                   uint32_t n_committees, uint32_t cps_prev, uint32_t cps_cur, const uint8_t* chain_roots, const uint8_t* justified80,
                                   const uint8_t* domains64, uint32_t slots_per_epoch, uint32_t min_inclusion_delay, uint64_t effective_balance_increment,
                                   uint64_t base_reward_per_increment, int32_t* status_out, uint8_t* flag_mask_out, uint64_t* numerator_out,
                                   int32_t* block_status_out, uint32_t* block_first_out, uint64_t* block_reward_out, uint32_t* n_applied_out) {
    const char* what = f.what();
    int rc;
    if ((rc = check_block_attestations(ctx, what, wire, woff, n_att, block_off, block_slot, n_blocks, members, off, n_committees, cps_prev, cps_cur,
                                       chain_roots, justified80, domains64, slots_per_epoch, min_inclusion_delay, effective_balance_increment, status_out,
                                       flag_mask_out, numerator_out, block_status_out, block_first_out, block_reward_out, n_applied_out)) ||
        (rc = check_wire(ctx, woff, n_att, wire_len, what)) || (rc = check_offsets(ctx, block_off, n_blocks, what, "block_off")))
        return rc;
    if (block_off[n_blocks] != n_att) return reject(ctx, what, "block_off must end at n_att");
    const uint64_t e = block_slot[0] / slots_per_epoch;
    if (block_slot[0] >= (1ull << 63)) return reject(ctx, what, "block slot out of range");
    for (uint32_t b = 1; b < n_blocks; b++)
        if (block_slot[b] <= block_slot[b - 1] || block_slot[b] / slots_per_epoch != e)
            return reject(ctx, what, "block slots must increase strictly and lie in one epoch");
    if (e > 0 ? cps_prev == 0 : cps_prev != 0) return reject(ctx, what, "cps_prev must be 0 exactly at epoch 0");
    if (f.electra) {
        if ((rc = check_offsets(ctx, off, n_committees, what))) return rc;
        // the largest member count of one slot's committees: the slots of e - 1 (cps_prev rows each), then those of e (cps_cur rows each)
        f.row_max = 1;
        for (uint32_t s = 0; s < 2 * slots_per_epoch; s++) {
            const uint32_t cps = s < slots_per_epoch ? cps_prev : cps_cur;
            const uint32_t c = s < slots_per_epoch ? s * cps_prev : cps_prev * slots_per_epoch + (s - slots_per_epoch) * cps_cur;
            f.row_max = std::max(f.row_max, off[c + cps] - off[c]);
        }
    }
    if ((rc = check_ba_shape(ctx, n_att, f)) || (!f.electra && (rc = check_committees(ctx, off, n_committees, f.bits_stride, what)))) return rc;
    const uint64_t n_sig = off[n_committees];
    CK(cudaSetDevice(ctx->device));
    staging st(ctx);
    const uint8_t* dwire = st.in(wire, wire_len, 16);
    const uint32_t* dwoff = st.in(woff, (size_t)n_att + 1);
    const uint32_t* dboff = st.in(block_off, (size_t)n_blocks + 1);
    const uint64_t* dbslot = st.in(block_slot, n_blocks);
    const uint32_t* dmem = st.in(members, n_sig, 4);
    const uint32_t* doff = st.in(off, (size_t)n_committees + 1);
    const uint8_t* droots = st.in(chain_roots, 64ull * slots_per_epoch);
    int32_t* dst = st.out(status_out, n_att);
    uint8_t* dmask = st.out(flag_mask_out, n_att);
    uint64_t* dnum = st.out(numerator_out, n_att);
    int32_t* dbst = st.out(block_status_out, n_blocks);
    uint32_t* dbfirst = st.out(block_first_out, n_blocks);
    uint64_t* dbrew = st.out(block_reward_out, n_blocks);
    uint32_t* dnapp = st.out(n_applied_out, 1);
    if (st.rc) return st.rc;
    if ((rc = block_attestations_enqueue(ctx, f, dwire, wire_len, dwoff, n_att, dboff, dbslot, n_blocks, dmem, doff, n_sig, cps_prev, cps_cur, droots,
                                         justified80, domains64, slots_per_epoch, min_inclusion_delay, effective_balance_increment,
                                         base_reward_per_increment, dst, dmask, dnum, dbst, dbfirst, dbrew, dnapp, ctx->s_main)))
        return rc;
    return st.finish();
}
int b2_block_attestations(b2_ctx* ctx, const uint8_t* wire, uint64_t wire_len, const uint32_t* woff, uint32_t n_att, const uint32_t* block_off,
                          const uint64_t* block_slot, uint32_t n_blocks, const uint32_t* members, const uint32_t* off, uint32_t n_committees, uint32_t cps_prev,
                          uint32_t cps_cur, const uint8_t* chain_roots, const uint8_t* justified80, const uint8_t* domains64, uint32_t slots_per_epoch,
                          uint32_t min_inclusion_delay, uint32_t bits_stride, uint64_t effective_balance_increment, uint64_t base_reward_per_increment,
                          int32_t* status_out, uint8_t* flag_mask_out, uint64_t* numerator_out, int32_t* block_status_out, uint32_t* block_first_out,
                          uint64_t* block_reward_out, uint32_t* n_applied_out) {
    B2_NVTX;
    return block_attestations_host(ctx, {false, bits_stride, 0, 0, 0}, wire, wire_len, woff, n_att, block_off, block_slot, n_blocks, members, off,
                                   n_committees, cps_prev, cps_cur, chain_roots, justified80, domains64, slots_per_epoch, min_inclusion_delay,
                                   effective_balance_increment, base_reward_per_increment, status_out, flag_mask_out, numerator_out, block_status_out,
                                   block_first_out, block_reward_out, n_applied_out);
}
int b2_block_attestations_electra(b2_ctx* ctx, const uint8_t* wire, uint64_t wire_len, const uint32_t* woff, uint32_t n_att, const uint32_t* block_off,
                                  const uint64_t* block_slot, uint32_t n_blocks, const uint32_t* members, const uint32_t* off, uint32_t n_committees,
                                  uint32_t cps_prev, uint32_t cps_cur, const uint8_t* chain_roots, const uint8_t* justified80, const uint8_t* domains64,
                                  uint32_t slots_per_epoch, uint32_t min_inclusion_delay, uint32_t max_committees_per_slot,
                                  uint32_t max_validators_per_committee, uint64_t effective_balance_increment, uint64_t base_reward_per_increment,
                                  int32_t* status_out, uint8_t* flag_mask_out, uint64_t* numerator_out, int32_t* block_status_out,
                                  uint32_t* block_first_out, uint64_t* block_reward_out, uint32_t* n_applied_out) {
    B2_NVTX;
    return block_attestations_host(ctx, {true, 0, max_committees_per_slot, max_validators_per_committee, 0}, wire, wire_len, woff, n_att, block_off,
                                   block_slot, n_blocks, members, off, n_committees, cps_prev, cps_cur, chain_roots, justified80, domains64,
                                   slots_per_epoch, min_inclusion_delay, effective_balance_increment, base_reward_per_increment, status_out, flag_mask_out,
                                   numerator_out, block_status_out, block_first_out, block_reward_out, n_applied_out);
}

// ------------------------------------------------------------------------------------------ sync committee messages (syncmsg.cuh)
// SyncCommitteeMessage (pos-evolution.md:548-557) through the sync_committee_{subnet_id} checks of the upstream Altair p2p spec, and the
// accepted ones into the SyncCommitteeContributions and SyncAggregates of process_sync_committee_contributions (upstream Altair validator
// spec).  The signature check shares the AggregateVerify buffers with b2_aggregate_verify[_dev] and the intakes: one stream for all of them.
static int check_sync_committee_messages(b2_ctx* ctx, const void* wire, const void* woff, uint32_t n, const void* subnet, const void* position_validator,
                                         uint32_t committee_size, uint32_t subnet_count, const void* domain32, const void* status_out, const void* root_id_out,
                                         const void* roots32_out, const void* n_roots_out, const void* contrib_bits_out, const void* contrib_sig96_out,
                                         const void* contrib_present_out, const void* agg_bits_out, const void* agg_sig96_out) {
    REQUIRE(ctx && wire && woff && subnet && position_validator && domain32 && status_out && root_id_out && roots32_out && n_roots_out &&
                contrib_bits_out && contrib_sig96_out && contrib_present_out && agg_bits_out && agg_sig96_out && n > 0 && n < (1u << 24) &&
                committee_size > 0 && subnet_count > 0 && (uint64_t)n * (subnet_count + 1) < (1ull << 31),
            "sync_committee_messages: bad arguments");
    REQUIRE(committee_size % subnet_count == 0, "sync_committee_messages: committee_size must be a multiple of subnet_count");
    REQUIRE(committee_size <= B2_SYNC_MAX_SIZE, "sync_committee_messages: committee_size above the kernels' limit (1024)");
    return ctx->n_val > 0 ? B2_OK : reject(ctx, "sync_committee_messages", "registry not loaded");
}
int b2_sync_committee_messages_dev(b2_ctx* ctx, const uint8_t* d_wire, uint64_t wire_len, const uint32_t* d_woff, uint32_t n, const uint32_t* d_subnet,
                                   const uint32_t* d_position_validator, uint32_t committee_size, uint32_t subnet_count, uint64_t current_slot,
                                   const uint8_t* domain32, int32_t* d_status_out, uint32_t* d_root_id_out, uint8_t* d_roots32_out,
                                   uint32_t* d_n_roots_out, uint8_t* d_contrib_bits_out, uint8_t* d_contrib_sig96_out, uint8_t* d_contrib_present_out,
                                   uint8_t* d_agg_bits_out, uint8_t* d_agg_sig96_out, void* stream) {
    B2_NVTX;
    int rc;
    if ((rc = check_sync_committee_messages(ctx, d_wire, d_woff, n, d_subnet, d_position_validator, committee_size, subnet_count, domain32, d_status_out, d_root_id_out,
                                            d_roots32_out, d_n_roots_out, d_contrib_bits_out, d_contrib_sig96_out, d_contrib_present_out, d_agg_bits_out,
                                            d_agg_sig96_out)))
        return rc;
    CK(cudaSetDevice(ctx->device));
    const uint32_t sub = committee_size / subnet_count;
    const uint64_t nc = (uint64_t)n * subnet_count;
    uint32_t tab = 1;
    while (tab < 2 * n) tab <<= 1;
    scm_args A = {};
    A.wire = d_wire;
    A.wire_len = wire_len;
    A.woff = d_woff;
    A.n = n;
    A.subnet = d_subnet;
    A.pos_val = d_position_validator;
    A.size = committee_size;
    A.subnets = subnet_count;
    A.sub = sub;
    A.sb = (sub + 7) / 8;
    A.ab = (committee_size + 7) / 8;
    A.current_slot = current_slot;
    A.n_val = ctx->n_val;
    memcpy(A.dom.b, domain32, 32);
    A.rtab_mask = tab - 1;
    A.status = d_status_out;
    A.root_id = d_root_id_out;
    A.n_roots = d_n_roots_out;
    A.roots32 = d_roots32_out;
    A.cbits = d_contrib_bits_out;
    A.cpresent = d_contrib_present_out;
    A.abits = d_agg_bits_out;
    A.guard = ctx->d_guard;
    // the AggregateVerify verdicts (read by the kernels through A.ok); the decompressed item signatures, the gathered ones and the segment sums
    uint8_t *ok, *st, *gst;
    uint32_t *aff, *gaff, *sumjac;
    int32_t* segst;
    scratch sc(ctx, ctx->scm);
    sc(A.keys, committee_size); sc(A.canon, n); sc(A.first, committee_size); sc(A.pitem, committee_size); sc(A.proot, committee_size);
    sc(A.signer, n); sc(A.pair_off, (size_t)n + 1); sc(A.msg, (size_t)n * 32); sc(A.sig, (size_t)n * 96); sc(ok, n);
    sc(A.slot_of, n); sc(A.rtab, tab); sc(A.rmin, tab); sc(A.rid, n); sc(A.seg_off, nc + 1); sc(A.agg_off, (size_t)n + 1); sc(A.gsrc, committee_size);
    sc(aff, (size_t)n * 48, 16); sc(st, n, 16); sc(gaff, (size_t)committee_size * 48, 16); sc(gst, committee_size, 16);
    sc(sumjac, (nc + n) * 72); sc(segst, nc + n);
    if (sc.rc) return sc.rc;
    A.ok = ok;
    cudaStream_t s = (cudaStream_t)stream;
    CK(cudaMemsetAsync(A.first, 0xff, (size_t)committee_size * 4, s));
    CK(cudaMemsetAsync(A.rtab, 0xff, (size_t)tab * 4, s));
    CK(cudaMemsetAsync(A.rmin, 0xff, (size_t)tab * 4, s));
    k_scm_index<<<1, 1024, 0, s>>>(A);
    CKL(ctx);
    k_scm_parse<<<blocks_for(n, 128), 128, 0, s>>>(A);
    CKL(ctx);
    if ((rc = aggregate_verify_enqueue(ctx, A.signer, nullptr, A.msg, A.pair_off, n, A.sig, n, ok, s))) return rc;
    k_scm_first<<<blocks_for(n, 128), 128, 0, s>>>(A);
    CKL(ctx);
    k_scm_accept<<<blocks_for(n, 128), 128, 0, s>>>(A);
    CKL(ctx);
    k_scm_number<<<1, 1024, 0, s>>>(A);
    CKL(ctx);
    k_scm_positions<<<blocks_for(committee_size, 128), 128, 0, s>>>(A);
    CKL(ctx);
    k_scm_rows<<<blocks_for(nc + n, 128), 128, 0, s>>>(A);
    CKL(ctx);
    k_intake_scan<<<1, 1024, 0, s>>>(A.seg_off, (uint32_t)nc, nullptr);     // seg_off[nc] = the set positions of every root
    CKL(ctx);
    k_scm_gather<<<blocks_for(std::max<uint64_t>(committee_size, (uint64_t)n + 1), 128), 128, 0, s>>>(A);
    CKL(ctx);
    // bls.Aggregate of each contribution's and each root's signatures: the item signatures decompressed once (an item that was not
    // accepted holds zero bytes and is never gathered), gathered per set position, one segment per (root, subnet) and one per root
    k_g2_decompress<<<blocks_for(n, ctx->dec_block), ctx->dec_block, 0, s>>>(A.sig, n, aff, st);
    CKL(ctx);
    k_pack_gather<<<blocks_for(committee_size, 128), 128, 0, s>>>(aff, st, A.gsrc, A.seg_off + nc, gaff, gst);
    CKL(ctx);
    k_g2_segment_sum<<<(unsigned)nc, 32, 0, s>>>(gaff, gst, A.seg_off, (uint32_t)nc, sumjac, segst, committee_size, ctx->d_guard);
    CKL(ctx);
    k_g2_segment_sum<<<n, 32, 0, s>>>(gaff, gst, A.agg_off, n, sumjac + 72 * nc, segst + nc, committee_size, ctx->d_guard);
    CKL(ctx);
    k_g2_finish<<<blocks_for(nc, 32), 32, 0, s>>>(sumjac, segst, (uint32_t)nc, d_contrib_sig96_out, nullptr, nullptr);
    CKL(ctx);
    k_g2_finish<<<blocks_for(n, 32), 32, 0, s>>>(sumjac + 72 * nc, segst + nc, n, d_agg_sig96_out, nullptr, nullptr);
    CKL(ctx);
    return B2_OK;
}

int b2_sync_committee_messages(b2_ctx* ctx, const uint8_t* wire, uint64_t wire_len, const uint32_t* woff, uint32_t n, const uint32_t* subnet,
                               const uint32_t* position_validator, uint32_t committee_size, uint32_t subnet_count, uint64_t current_slot,
                               const uint8_t* domain32, int32_t* status_out, uint32_t* root_id_out, uint8_t* roots32_out, uint32_t* n_roots_out,
                               uint8_t* contrib_bits_out, uint8_t* contrib_sig96_out, uint8_t* contrib_present_out, uint8_t* agg_bits_out,
                               uint8_t* agg_sig96_out) {
    B2_NVTX;
    int rc;
    if ((rc = check_sync_committee_messages(ctx, wire, woff, n, subnet, position_validator, committee_size, subnet_count, domain32, status_out, root_id_out, roots32_out,
                                            n_roots_out, contrib_bits_out, contrib_sig96_out, contrib_present_out, agg_bits_out, agg_sig96_out)) ||
        (rc = check_wire(ctx, woff, n, wire_len, "sync_committee_messages")))
        return rc;
    for (uint32_t p = 0; p < committee_size; p++)
        REQUIRE(position_validator[p] < ctx->n_val, "sync_committee_messages: a position_validator entry is outside the registry");
    CK(cudaSetDevice(ctx->device));
    const uint32_t sub = committee_size / subnet_count;
    const size_t nc = (size_t)n * subnet_count;
    staging st(ctx);
    const uint8_t* dwire = st.in(wire, wire_len, 16);
    const uint32_t* dwoff = st.in(woff, (size_t)n + 1);
    const uint32_t* dsub = st.in(subnet, n);
    const uint32_t* dpv = st.in(position_validator, committee_size);
    int32_t* dst = st.out(status_out, n);
    uint32_t* drid = st.out(root_id_out, n);
    uint8_t* droots = st.out(roots32_out, (size_t)n * 32);
    uint32_t* dnr = st.out(n_roots_out, 1);
    uint8_t* dcb = st.out(contrib_bits_out, nc * ((sub + 7) / 8));
    uint8_t* dcs = st.out(contrib_sig96_out, nc * 96);
    uint8_t* dcp = st.out(contrib_present_out, nc);
    uint8_t* dab = st.out(agg_bits_out, (size_t)n * ((committee_size + 7) / 8));
    uint8_t* das = st.out(agg_sig96_out, (size_t)n * 96);
    if (st.rc) return st.rc;
    if ((rc = b2_sync_committee_messages_dev(ctx, dwire, wire_len, dwoff, n, dsub, dpv, committee_size, subnet_count, current_slot, domain32, dst, drid,
                                             droots, dnr, dcb, dcs, dcp, dab, das, ctx->s_main)))
        return rc;
    return st.finish();
}

// ------------------------------------------------------------------------------------------ sync committee contributions (synccontrib.cuh)
// SignedContributionAndProof through the sync_committee_contribution_and_proof checks of the upstream Altair p2p spec, and each root's best
// contribution per subnet into its SyncAggregate (process_sync_committee_contributions, upstream Altair validator spec).  The signature checks
// share the AggregateVerify buffers and pipeline slot 0's verify buffers with the synchronous verify calls and the intakes: one stream for all.
static int check_sync_contribution_and_proof_intake(b2_ctx* ctx, const void* wire, const void* woff, uint32_t n, const void* position_validator,
                                                    uint32_t committee_size, uint32_t subnet_count, const void* domains96, uint32_t target_aggregators,
                                                    const void* status_out, const void* root_id_out, const void* roots32_out, const void* n_roots_out,
                                                    const void* best_out, const void* agg_bits_out, const void* agg_sig96_out) {
    REQUIRE(ctx && wire && woff && position_validator && domains96 && status_out && root_id_out && roots32_out && n_roots_out && best_out &&
                agg_bits_out && agg_sig96_out && n > 0 && n < (1u << 24) && committee_size > 0 && subnet_count > 0 &&
                (uint64_t)n * (subnet_count + 1) < (1ull << 31),
            "sync_contribution_and_proof_intake: bad arguments");
    REQUIRE(committee_size % subnet_count == 0, "sync_contribution_and_proof_intake: committee_size must be a multiple of subnet_count");
    REQUIRE(committee_size <= B2_SYNC_MAX_SIZE, "sync_contribution_and_proof_intake: committee_size above the kernels' limit (1024)");
    REQUIRE(target_aggregators > 0, "sync_contribution_and_proof_intake: target_aggregators must be positive");
    return ctx->n_val > 0 ? B2_OK : reject(ctx, "sync_contribution_and_proof_intake", "registry not loaded");
}
int b2_sync_contribution_and_proof_intake_dev(b2_ctx* ctx, const uint8_t* d_wire, uint64_t wire_len, const uint32_t* d_woff, uint32_t n,
                                              const uint32_t* d_position_validator, uint32_t committee_size, uint32_t subnet_count,
                                              uint64_t current_slot, const uint8_t* domains96, uint32_t target_aggregators, int32_t* d_status_out,
                                              uint32_t* d_root_id_out, uint8_t* d_roots32_out, uint32_t* d_n_roots_out, uint32_t* d_best_out,
                                              uint8_t* d_agg_bits_out, uint8_t* d_agg_sig96_out, void* stream) {
    B2_NVTX;
    int rc;
    if ((rc = check_sync_contribution_and_proof_intake(ctx, d_wire, d_woff, n, d_position_validator, committee_size, subnet_count, domains96,
                                                       target_aggregators, d_status_out, d_root_id_out, d_roots32_out, d_n_roots_out, d_best_out,
                                                       d_agg_bits_out, d_agg_sig96_out)))
        return rc;
    CK(cudaSetDevice(ctx->device));
    const uint32_t sub = committee_size / subnet_count, sb = (sub + 7) / 8;
    const uint64_t nc = (uint64_t)n * subnet_count;
    uint32_t tab = 1;
    while (tab < 2 * n) tab <<= 1;
    scc_args A = {};
    A.wire = d_wire;
    A.wire_len = wire_len;
    A.woff = d_woff;
    A.n = n;
    A.size = committee_size;
    A.subnets = subnet_count;
    A.sub = sub;
    A.sb = sb;
    A.sw = (sb + 3) / 4;
    A.ab = (committee_size + 7) / 8;
    A.target = target_aggregators;
    A.current_slot = current_slot;
    A.n_val = ctx->n_val;
    memcpy(A.dom_sync.b, domains96, 32);
    memcpy(A.dom_sel.b, domains96 + 32, 32);
    memcpy(A.dom_cap.b, domains96 + 64, 32);
    A.rtab_mask = tab - 1;
    A.status = d_status_out;
    A.root_id = d_root_id_out;
    A.best = d_best_out;
    A.abits = d_agg_bits_out;
    A.guard = ctx->d_guard;
    scm_args& M = A.M;
    // k_scm_number reads a root at scm_item + SCM_ROOT: a contribution's root lies 8 bytes further into the item than a message's
    M.wire = d_wire + (SCC_ROOT - SCM_ROOT);
    M.woff = d_woff;
    M.n = n;
    M.pos_val = d_position_validator;
    M.size = committee_size;
    M.subnets = subnet_count;
    M.sub = sub;
    M.n_val = ctx->n_val;
    M.status = d_status_out;
    M.root_id = d_root_id_out;
    M.n_roots = d_n_roots_out;
    M.roots32 = d_roots32_out;
    M.guard = ctx->d_guard;
    // the verify verdicts (read by the kernels through A); the decompressed item signatures, the gathered ones and the root sums
    uint8_t *av_ok, *fav_ok, *st, *gst;
    uint32_t *aff, *gaff, *sumjac;
    int32_t* segst;
    scratch sc(ctx, ctx->scc);
    sc(M.keys, committee_size); sc(A.subnet, n); sc(A.canon, n); sc(A.rslot, n); sc(A.rtab, tab); sc(A.bw, (size_t)n * A.sw); sc(A.ones, n);
    sc(A.av_signer, 2 * (size_t)n); sc(A.av_off, 2 * (size_t)n + 1); sc(A.av_msg, (size_t)n * 64); sc(A.av_sig, (size_t)n * 192); sc(av_ok, 2 * (size_t)n);
    sc(A.members, (size_t)n * sub); sc(A.item_off, (size_t)n + 1); sc(A.fbits, (size_t)n * sb, 16); sc(A.fmsg, (size_t)n * 32); sc(A.fsig, (size_t)n * 96);
    sc(fav_ok, n); sc(A.taken, committee_size); sc(A.acc, committee_size); sc(M.slot_of, n); sc(M.rmin, tab); sc(M.rid, n);
    sc(A.bestkey, nc); sc(A.cnt, (size_t)n + 1); sc(A.gsrc, n);
    sc(aff, (size_t)n * 48, 16); sc(st, n, 16); sc(gaff, (size_t)n * 48, 16); sc(gst, n, 16); sc(sumjac, (size_t)n * 72); sc(segst, n);
    if (sc.rc) return sc.rc;
    A.av_ok = av_ok;
    A.fav_ok = fav_ok;
    cudaStream_t s = (cudaStream_t)stream;
    CK(cudaMemsetAsync(A.rtab, 0xff, (size_t)tab * 4, s));
    CK(cudaMemsetAsync(M.rmin, 0xff, (size_t)tab * 4, s));
    CK(cudaMemsetAsync(A.taken, 0, committee_size, s));
    CK(cudaMemsetAsync(A.bestkey, 0, nc * 8, s));
    k_scm_index<<<1, 1024, 0, s>>>(M);
    CKL(ctx);
    k_scc_parse<<<blocks_for(n, 64), 64, 0, s>>>(A);
    CKL(ctx);
    // FastAggregateVerify of the contributions over their subnets' member rows, then AggregateVerify of the 2n single-key sets
    pk_source P = {A.members, A.item_off, A.fbits, sb, nullptr, 0};
    if ((rc = verify_fork(ctx, ctx->slot[0], P, A.fmsg, n, s)) || (rc = verify_main(ctx, ctx->slot[0], A.fsig, n, fav_ok, s))) return rc;
    if ((rc = aggregate_verify_enqueue(ctx, A.av_signer, nullptr, A.av_msg, A.av_off, 2ull * n, A.av_sig, 2 * n, av_ok, s))) return rc;
    k_scc_order<<<subnet_count, 32, 0, s>>>(A);
    CKL(ctx);
    k_scc_claim<<<blocks_for(n, 128), 128, 0, s>>>(A);
    CKL(ctx);
    k_scm_number<<<1, 1024, 0, s>>>(M);
    CKL(ctx);
    k_scc_best<<<blocks_for(n, 128), 128, 0, s>>>(A);
    CKL(ctx);
    k_scc_rows<<<blocks_for(n, 128), 128, 0, s>>>(A);
    CKL(ctx);
    k_intake_scan<<<1, 1024, 0, s>>>(A.cnt, n, nullptr);      // cnt[n] = the best items of every root
    CKL(ctx);
    k_scc_gather<<<blocks_for(n, 128), 128, 0, s>>>(A);
    CKL(ctx);
    // bls.Aggregate of each root's best contributions: the item signatures decompressed once (an item that was not accepted holds zero
    // bytes and is never gathered), gathered in (root, subnet) order, one segment per root
    k_g2_decompress<<<blocks_for(n, ctx->dec_block), ctx->dec_block, 0, s>>>(A.fsig, n, aff, st);
    CKL(ctx);
    k_pack_gather<<<blocks_for(n, 128), 128, 0, s>>>(aff, st, A.gsrc, A.cnt + n, gaff, gst);
    CKL(ctx);
    k_g2_segment_sum<<<n, 32, 0, s>>>(gaff, gst, A.cnt, n, sumjac, segst, n, ctx->d_guard);
    CKL(ctx);
    k_g2_finish<<<blocks_for(n, 32), 32, 0, s>>>(sumjac, segst, n, d_agg_sig96_out, nullptr, nullptr);
    CKL(ctx);
    return B2_OK;
}

int b2_sync_contribution_and_proof_intake(b2_ctx* ctx, const uint8_t* wire, uint64_t wire_len, const uint32_t* woff, uint32_t n,
                                          const uint32_t* position_validator, uint32_t committee_size, uint32_t subnet_count, uint64_t current_slot,
                                          const uint8_t* domains96, uint32_t target_aggregators, int32_t* status_out, uint32_t* root_id_out,
                                          uint8_t* roots32_out, uint32_t* n_roots_out, uint32_t* best_out, uint8_t* agg_bits_out,
                                          uint8_t* agg_sig96_out) {
    B2_NVTX;
    int rc;
    if ((rc = check_sync_contribution_and_proof_intake(ctx, wire, woff, n, position_validator, committee_size, subnet_count, domains96, target_aggregators,
                                                       status_out, root_id_out, roots32_out, n_roots_out, best_out, agg_bits_out, agg_sig96_out)) ||
        (rc = check_wire(ctx, woff, n, wire_len, "sync_contribution_and_proof_intake")))
        return rc;
    for (uint32_t p = 0; p < committee_size; p++)
        REQUIRE(position_validator[p] < ctx->n_val, "sync_contribution_and_proof_intake: a position_validator entry is outside the registry");
    CK(cudaSetDevice(ctx->device));
    staging st(ctx);
    const uint8_t* dwire = st.in(wire, wire_len, 16);
    const uint32_t* dwoff = st.in(woff, (size_t)n + 1);
    const uint32_t* dpv = st.in(position_validator, committee_size);
    int32_t* dst = st.out(status_out, n);
    uint32_t* drid = st.out(root_id_out, n);
    uint8_t* droots = st.out(roots32_out, (size_t)n * 32);
    uint32_t* dnr = st.out(n_roots_out, 1);
    uint32_t* dbest = st.out(best_out, (size_t)n * subnet_count);
    uint8_t* dab = st.out(agg_bits_out, (size_t)n * ((committee_size + 7) / 8));
    uint8_t* das = st.out(agg_sig96_out, (size_t)n * 96);
    if (st.rc) return st.rc;
    if ((rc = b2_sync_contribution_and_proof_intake_dev(ctx, dwire, wire_len, dwoff, n, dpv, committee_size, subnet_count, current_slot, domains96,
                                                        target_aggregators, dst, drid, droots, dnr, dbest, dab, das, ctx->s_main)))
        return rc;
    return st.finish();
}

// ------------------------------------------------------------------------------------------ committee shuffle
static int check_shuffle_committees(b2_ctx* ctx, const uint8_t* seed32, const uint32_t* members_out, uint32_t rounds) {
    REQUIRE(ctx && seed32 && members_out && rounds <= 255, "shuffle_committees: bad arguments");
    return B2_OK;
}
int b2_shuffle_committees_dev(b2_ctx* ctx, const uint8_t* d_seed32, const uint32_t* d_active, uint32_t n_active, uint32_t rounds,
                              uint32_t* d_members_out, void* stream) {
    B2_NVTX;
    int rc;
    if ((rc = check_shuffle_committees(ctx, d_seed32, d_members_out, rounds))) return rc;
    if (n_active == 0) return B2_OK;
    CK(cudaSetDevice(ctx->device));
    cudaStream_t s = (cudaStream_t)stream;
    const uint32_t nblk = (n_active + 255) / 256;
    if ((rc = ensure(ctx, ctx->sc_shuf, (size_t)rounds * nblk * 32 + 16)) || (rc = ensure(ctx, ctx->sc_pivot, (size_t)rounds * 8 + 16))) return rc;
    if (rounds) {
        k_shuffle_sources<<<blocks_for((uint64_t)rounds * (nblk + 1), 128), 128, 0, s>>>(d_seed32, n_active, rounds, nblk, (uint8_t*)ctx->sc_shuf.p,
                                                                                  (unsigned long long*)ctx->sc_pivot.p);
        CKL(ctx);
    }
    k_shuffle_apply<<<blocks_for(n_active, 256), 256, 0, s>>>(n_active, rounds, nblk, (const uint8_t*)ctx->sc_shuf.p,
                                                             (const unsigned long long*)ctx->sc_pivot.p, d_active, d_members_out);
    CKL(ctx);
    return B2_OK;
}

int b2_shuffle_committees(b2_ctx* ctx, const uint8_t* seed32, const uint32_t* active, uint32_t n_active, uint32_t rounds, uint32_t* members_out) {
    B2_NVTX;
    int rc;
    if ((rc = check_shuffle_committees(ctx, seed32, members_out, rounds))) return rc;
    if (n_active == 0) return B2_OK;
    CK(cudaSetDevice(ctx->device));
    staging st(ctx);
    const uint8_t* dseed = st.in(seed32, 32);
    const uint32_t* dact = active ? st.in(active, n_active) : nullptr;
    uint32_t* dm = st.out(members_out, n_active);
    if ((rc = st.rc) || (rc = b2_shuffle_committees_dev(ctx, dseed, dact, n_active, rounds, dm, ctx->s_main))) return rc;
    return st.finish();
}

// ------------------------------------------------------------------------------------------ latest messages
int b2_latest_messages_reset(b2_ctx* ctx) {
    B2_NVTX;
    REQUIRE(ctx && ctx->n_val > 0, "latest_messages_reset: registry not loaded");
    CK(cudaSetDevice(ctx->device));
    CK(cudaMemsetAsync(ctx->reg.lmd_key, 0, ctx->n_val * 8, ctx->s_main));
    CK(cudaMemsetAsync(ctx->reg.lmd_block, 0, ctx->n_val * 4, ctx->s_main));
    CK(cudaMemsetAsync(ctx->reg.equiv, 0, ctx->n_val, ctx->s_main));
    CK(cudaStreamSynchronize(ctx->s_main));
    return B2_OK;
}

int b2_latest_messages_load(b2_ctx* ctx, const uint64_t* epoch, const uint32_t* block_idx, const uint8_t* has_msg, const uint8_t* equivocating,
                            uint64_t n) {
    B2_NVTX;
    REQUIRE(ctx && epoch && block_idx && has_msg && equivocating && n == ctx->n_val && n > 0, "latest_messages_load: bad arguments / registry size");
    std::vector<unsigned long long> key(n);
    for (uint64_t v = 0; v < n; v++) {
        REQUIRE(!has_msg[v] || epoch[v] < 0xffffffffull, "latest_messages_load: epoch does not fit 32 bits");
        key[v] = has_msg[v] ? ((epoch[v] << 32) | 0xffffffffull) : 0ull;
    }
    CK(cudaSetDevice(ctx->device));
    cudaStream_t s = ctx->s_main;
    CK(cudaMemcpyAsync(ctx->reg.lmd_key, key.data(), n * 8, cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync(ctx->reg.lmd_block, block_idx, n * 4, cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync(ctx->reg.equiv, equivocating, n, cudaMemcpyHostToDevice, s));
    CK(cudaStreamSynchronize(s));
    return B2_OK;
}

int b2_latest_messages_read(b2_ctx* ctx, uint64_t* epoch, uint32_t* block_idx, uint8_t* has_msg, uint64_t n) {
    B2_NVTX;
    REQUIRE(ctx && epoch && block_idx && has_msg && n == ctx->n_val && n > 0, "latest_messages_read: bad arguments / registry size");
    std::vector<unsigned long long> key(n);
    CK(cudaSetDevice(ctx->device));
    staging st(ctx);
    st.out(key.data(), ctx->reg.lmd_key, n);
    st.out(block_idx, ctx->reg.lmd_block, n);
    int rc;
    if ((rc = st.finish())) return rc;
    for (uint64_t v = 0; v < n; v++) {
        has_msg[v] = key[v] != 0;
        epoch[v] = key[v] >> 32;
        if (!has_msg[v]) block_idx[v] = 0;
    }
    return B2_OK;
}

static int check_latest_messages_update(b2_ctx* ctx, const void* members, const void* off, const void* bits, uint32_t bits_stride, const void* target_epoch,
                                        const void* block_idx, uint32_t n_agg) {
    REQUIRE(ctx && members && off && bits && target_epoch && block_idx && n_agg > 0 && bits_stride > 0, "latest_messages_update: bad arguments");
    return ctx->n_val > 0 ? B2_OK : reject(ctx, "latest_messages_update", "registry not loaded");
}
int b2_latest_messages_update_dev(b2_ctx* ctx, const uint32_t* d_members, const uint32_t* d_off, const uint8_t* d_bits, uint32_t bits_stride,
                                  const uint64_t* d_target_epoch, const uint32_t* d_block_idx, const uint8_t* d_accept, uint32_t n_agg, void* stream) {
    B2_NVTX;
    int rc;
    if ((rc = check_latest_messages_update(ctx, d_members, d_off, d_bits, bits_stride, d_target_epoch, d_block_idx, n_agg))) return rc;
    CK(cudaSetDevice(ctx->device));
    cudaStream_t s = (cudaStream_t)stream;
    k_lmd_phase1<<<n_agg, 128, 0, s>>>(d_members, d_off, d_bits, bits_stride, d_target_epoch, d_accept, ctx->reg.equiv, n_agg, ctx->reg.lmd_key,
                                       ctx->n_val, ctx->d_guard);
    CKL(ctx);
    k_lmd_phase2<<<n_agg, 128, 0, s>>>(d_members, d_off, d_bits, bits_stride, d_target_epoch, d_block_idx, d_accept, ctx->reg.equiv, n_agg,
                                       ctx->reg.lmd_key, ctx->reg.lmd_block, ctx->n_val);
    CKL(ctx);
    return B2_OK;
}

int b2_latest_messages_update(b2_ctx* ctx, const uint32_t* members, const uint32_t* off, const uint8_t* bits, uint32_t bits_stride,
                              const uint64_t* target_epoch, const uint32_t* block_idx, const uint8_t* accept, uint32_t n_agg) {
    B2_NVTX;
    int rc;
    if ((rc = check_latest_messages_update(ctx, members, off, bits, bits_stride, target_epoch, block_idx, n_agg)) ||
        (rc = check_batch(ctx, members, off, bits_stride, n_agg, ctx->n_val, "latest_messages_update")))
        return rc;
    for (uint32_t a = 0; a < n_agg; a++) REQUIRE(target_epoch[a] < 0xffffffffull, "latest_messages_update: epoch does not fit 32 bits");
    CK(cudaSetDevice(ctx->device));
    staging st(ctx);
    const uint32_t* dm = st.in(members, off[n_agg], 4);
    const uint32_t* dof = st.in(off, (size_t)n_agg + 1);
    const uint8_t* db = st.in(bits, (size_t)n_agg * bits_stride, 16);
    const uint64_t* dte = st.in(target_epoch, n_agg);
    const uint32_t* dbi = st.in(block_idx, n_agg);
    const uint8_t* dacc = accept ? st.in(accept, n_agg) : nullptr;
    if ((rc = st.rc) || (rc = b2_latest_messages_update_dev(ctx, dm, dof, db, bits_stride, dte, dbi, dacc, n_agg, ctx->s_main))) return rc;
    return st.finish();
}

// ------------------------------------------------------------------------------------------ participation flags (process_attestation :738-754)
int b2_participation_load(b2_ctx* ctx, int which, const uint8_t* participation, uint64_t n) {
    B2_NVTX;
    REQUIRE(ctx && (which == 0 || which == 1) && participation && n == ctx->n_val && n > 0, "participation_load: bad arguments / registry size");
    CK(cudaSetDevice(ctx->device));
    int rc;
    const size_t words = (n + 3) / 4;
    // tables allocated by this call join the context only once they are initialised
    dbuf part, first;
    if (!ctx->reg.part[which] && (rc = ensure(ctx, part, words * 4))) return rc;
    if (!ctx->reg.part_first) {
        if ((rc = ensure(ctx, first, 3 * n * 4))) return rc;
        CK(cudaMemsetAsync(first, 0xff, 3 * n * 4, ctx->s_main));
    }
    void* dst = part ? part : ctx->reg.part[which];
    CK(cudaMemsetAsync(dst, 0, words * 4, ctx->s_main));
    CK(cudaMemcpyAsync(dst, participation, n, cudaMemcpyHostToDevice, ctx->s_main));
    CK(cudaStreamSynchronize(ctx->s_main));
    if (part) ctx->reg.part[which] = std::move(part);
    if (first) ctx->reg.part_first = std::move(first);
    return B2_OK;
}
int b2_participation_read(b2_ctx* ctx, int which, uint8_t* participation_out, uint64_t n) {
    B2_NVTX;
    REQUIRE(ctx && (which == 0 || which == 1) && participation_out && n == ctx->n_val && ctx->reg.part[which], "participation_read: not loaded / bad arguments");
    CK(cudaSetDevice(ctx->device));
    staging st(ctx);
    st.out(participation_out, ctx->reg.part[which], n);
    return st.finish();
}
int b2_participation_update(b2_ctx* ctx, int which, const uint32_t* members, const uint32_t* off, const uint8_t* bits, uint32_t bits_stride,
                            const uint8_t* flag_mask, const uint8_t* accept, uint32_t n_agg, uint64_t effective_balance_increment,
                            uint64_t base_reward_per_increment, uint64_t* numerator_out) {
    B2_NVTX;
    REQUIRE(ctx && (which == 0 || which == 1) && members && off && bits && flag_mask && numerator_out && n_agg > 0 && bits_stride > 0 &&
                effective_balance_increment > 0, "participation_update: bad arguments");
    REQUIRE(ctx->n_val > 0 && ctx->reg.part[which], "participation_update: registry / participation table not loaded");
    int rc;
    if ((rc = check_batch(ctx, members, off, bits_stride, n_agg, ctx->n_val, "participation_update"))) return rc;
    CK(cudaSetDevice(ctx->device));
    cudaStream_t s = ctx->s_main;
    staging st(ctx);
    const uint32_t* dm = st.in(members, off[n_agg], 4);
    const uint32_t* dof = st.in(off, (size_t)n_agg + 1);
    const uint8_t* db = st.in(bits, (size_t)n_agg * bits_stride, 16);
    const uint8_t* dmask = st.in(flag_mask, n_agg);
    const uint8_t* dacc = accept ? st.in(accept, n_agg) : nullptr;
    uint64_t* dnum = st.out(numerator_out, n_agg);
    if (st.rc) return st.rc;
    const registry_tables& R = ctx->reg;
    k_part_phase1<<<n_agg, 128, 0, s>>>(dm, dof, db, bits_stride, dmask, dacc, n_agg, R.part[which], R.part_first);
    CKL(ctx);
    k_part_phase2<<<n_agg, 128, 0, s>>>(dm, dof, db, bits_stride, dmask, dacc, n_agg, R.part_first, R.eff, effective_balance_increment,
                                        base_reward_per_increment, (unsigned long long*)dnum);
    CKL(ctx);
    k_part_phase3<<<n_agg, 128, 0, s>>>(dm, dof, db, bits_stride, dmask, dacc, n_agg, R.part_first, R.part[which]);
    CKL(ctx);
    return st.finish();
}

// ------------------------------------------------------------------------------------------ FFG balance sums (:793-803)
int b2_ffg_balances(b2_ctx* ctx, uint32_t flag_index, uint64_t* out4) {
    B2_NVTX;
    REQUIRE(ctx && out4 && flag_index < 8, "ffg_balances: bad arguments");
    REQUIRE(ctx->n_val > 0, "ffg_balances: registry not loaded");
    CK(cudaSetDevice(ctx->device));
    cudaStream_t s = ctx->s_main;
    staging st(ctx);
    uint64_t* d4 = st.out(out4, 4);
    if (st.rc) return st.rc;
    CK(cudaMemsetAsync(d4, 0, 32, s));
    k_ffg_balances<<<ctx->n_sm * 4, 256, 0, s>>>(ctx->n_val, ctx->reg.eff, ctx->reg.flags, ctx->reg.part[0], ctx->reg.part[1], flag_index,
                                                 (unsigned long long*)d4);
    CKL(ctx);
    return st.finish();
}

// ------------------------------------------------------------------------------------------ fork-choice variants
int b2_set_fork_choice_params(b2_ctx* ctx, uint64_t min_vote_epoch, int exclude_slashed) {
    B2_NVTX;
    REQUIRE(ctx && min_vote_epoch < 0xffffffffull, "set_fork_choice_params: bad arguments");
    ctx->fc_min_key = (unsigned long long)min_vote_epoch << 32;
    ctx->fc_exclude_slashed = exclude_slashed ? 1 : 0;
    return B2_OK;
}

int b2_set_verify_mode(b2_ctx* ctx, int mode, const uint8_t* seed32) {
    B2_NVTX;
    REQUIRE(ctx && (mode == 0 || (mode == 1 && seed32)), "set_verify_mode: bad arguments (mode 1 needs a 32-byte seed)");
    CK(cudaSetDevice(ctx->device));
    CK(cudaDeviceSynchronize());                   // no epoch in flight may see the mode change half way
    if (mode == 1) CK(cudaMemcpy(ctx->d_rlc_seed, seed32, 32, cudaMemcpyHostToDevice));
    ctx->verify_mode = mode;
    return B2_OK;
}

int b2_on_attester_slashing(b2_ctx* ctx, const uint32_t* indices_1, uint32_t n1, const uint32_t* indices_2, uint32_t n2) {
    B2_NVTX;
    REQUIRE(ctx && ctx->n_val > 0 && (n1 == 0 || indices_1) && (n2 == 0 || indices_2), "on_attester_slashing: bad arguments / registry not loaded");
    for (uint32_t i = 1; i < n1; i++) REQUIRE(indices_1[i - 1] < indices_1[i], "on_attester_slashing: attesting_indices must be sorted and unique");
    for (uint32_t i = 1; i < n2; i++) REQUIRE(indices_2[i - 1] < indices_2[i], "on_attester_slashing: attesting_indices must be sorted and unique");
    if (n1 == 0 || n2 == 0) return B2_OK;
    CK(cudaSetDevice(ctx->device));
    staging st(ctx);
    const uint32_t* d1 = st.in(indices_1, n1);
    const uint32_t* d2 = st.in(indices_2, n2);
    if (st.rc) return st.rc;
    k_mark_equivocating<<<blocks_for(n1, 128), 128, 0, ctx->s_main>>>(d1, n1, d2, n2, ctx->n_val, ctx->reg.equiv);
    CKL(ctx);
    return st.finish();
}

// ------------------------------------------------------------------------------------------ slasher (is_slashable_attestation_data :1128-1143)
static slasher_view slasher_view_of(const slasher_tables& t) {
    return {t.min_span, t.max_span, t.first_id, t.count, t.root, t.n_val, t.n_rows, t.v_begin, t.H, t.K, t.cur, t.cur >= t.H - 1 ? t.cur - (t.H - 1) : 0};
}
// every column empty
static int slasher_clear(b2_ctx* ctx, const slasher_tables& t, cudaStream_t s) {
    const size_t table = (size_t)t.n_rows * t.H * 2;
    CK(cudaMemsetAsync(t.min_span, 0xff, table, s));
    CK(cudaMemsetAsync(t.max_span, 0, table, s));
    CK(cudaMemsetAsync(t.first_id, 0xff, table, s));
    CK(cudaMemsetAsync(t.count, 0, (size_t)t.H * 4, s));
    return B2_OK;
}

int b2_slasher_init_range(b2_ctx* ctx, uint64_t n_validators, uint64_t v_begin, uint64_t v_end, uint32_t history_epochs,
                          uint32_t max_attestations_per_target, uint64_t current_epoch) {
    B2_NVTX;
    // the bounds keep the byte count below 2^52: no 64-bit overflow
    REQUIRE(ctx && n_validators > 0 && n_validators < (1ull << 32) && v_begin < v_end && v_end <= n_validators && history_epochs > 0 &&
                history_epochs <= 65535 && max_attestations_per_target > 0 && max_attestations_per_target <= 65535 && current_epoch < 0xffffffffull,
            "slasher_init: bad arguments (validators < 2^32, 0 <= v_begin < v_end <= validators, 1 <= history_epochs, "
            "max_attestations_per_target <= 65535, epoch < 2^32 - 1)");
    CK(cudaSetDevice(ctx->device));
    const uint64_t rows = v_end - v_begin;
    const uint64_t table = rows * history_epochs * 2, log = (uint64_t)history_epochs * max_attestations_per_target * 32;
    const uint64_t bytes = 3 * table + log + (uint64_t)history_epochs * 4;
    size_t free_b = 0, total_b = 0;
    CK(cudaMemGetInfo(&free_b, &total_b));
    if (bytes > free_b) {      // refused before any allocation is tried: the card may be shared
        snprintf(ctx->err, sizeof(ctx->err), "slasher_init: %llu bytes needed, %llu free on the device", (unsigned long long)bytes, (unsigned long long)free_b);
        return B2_ENOMEM;
    }
    slasher_tables t;      // built aside: a failed init leaves a previous slasher in place
    int rc;
    if ((rc = ensure(ctx, t.min_span, table)) || (rc = ensure(ctx, t.max_span, table)) || (rc = ensure(ctx, t.first_id, table)) ||
        (rc = ensure(ctx, t.root, log)) || (rc = ensure(ctx, t.count, (size_t)history_epochs * 4)))
        return rc;
    t.n_val = n_validators;
    t.n_rows = rows;
    t.v_begin = (uint32_t)v_begin;
    t.H = history_epochs;
    t.K = max_attestations_per_target;
    t.cur = (uint32_t)current_epoch;
    if ((rc = slasher_clear(ctx, t, ctx->s_main))) return rc;
    CK(cudaStreamSynchronize(ctx->s_main));
    ctx->sl = std::move(t);
    return B2_OK;
}

int b2_slasher_init(b2_ctx* ctx, uint64_t n_validators, uint32_t history_epochs, uint32_t max_attestations_per_target, uint64_t current_epoch) {
    return b2_slasher_init_range(ctx, n_validators, 0, n_validators, history_epochs, max_attestations_per_target, current_epoch);
}

int b2_slasher_free(b2_ctx* ctx) {
    B2_NVTX;
    REQUIRE(ctx, "null context");
    CK(cudaSetDevice(ctx->device));
    CK(cudaDeviceSynchronize());
    ctx->sl = slasher_tables();
    return B2_OK;
}

static int check_slasher_advance(b2_ctx* ctx, uint64_t current_epoch) {
    REQUIRE(ctx && ctx->sl.H, "slasher_advance: no slasher (b2_slasher_init)");
    return current_epoch >= ctx->sl.cur && current_epoch < 0xffffffffull ? B2_OK
                                                                         : reject(ctx, "slasher_advance", "the current epoch only moves forward and fits 32 bits");
}
int b2_slasher_advance_dev(b2_ctx* ctx, uint64_t current_epoch, void* stream) {
    B2_NVTX;
    int rc;
    if ((rc = check_slasher_advance(ctx, current_epoch))) return rc;
    slasher_tables& t = ctx->sl;
    if (current_epoch == t.cur) return B2_OK;
    CK(cudaSetDevice(ctx->device));
    cudaStream_t s = (cudaStream_t)stream;
    const uint64_t n_cols = current_epoch - t.cur;
    if (n_cols >= t.H) {
        if ((rc = slasher_clear(ctx, t, s))) return rc;
    } else {
        const unsigned blocks = (unsigned)std::min<uint64_t>((t.n_rows * n_cols + 255) / 256, (uint64_t)ctx->n_sm * 16);
        k_slasher_advance<<<blocks, 256, 0, s>>>(slasher_view_of(t), t.cur + 1, (uint32_t)n_cols);
        CKL(ctx);
    }
    t.cur = (uint32_t)current_epoch;      // the window of every update enqueued from now on; they are ordered after the reset by the caller
    return B2_OK;
}

int b2_slasher_advance(b2_ctx* ctx, uint64_t current_epoch) {
    B2_NVTX;
    int rc;
    if ((rc = check_slasher_advance(ctx, current_epoch))) return rc;
    if (current_epoch == ctx->sl.cur) return B2_OK;      // nothing to wait for
    CK(cudaSetDevice(ctx->device));
    CK(cudaDeviceSynchronize());      // updates enqueued on the caller's streams see the window they were enqueued with
    if ((rc = b2_slasher_advance_dev(ctx, current_epoch, ctx->s_main))) return rc;
    CK(cudaStreamSynchronize(ctx->s_main));
    return B2_OK;
}

static int check_slasher_update(b2_ctx* ctx, const void* members, const void* off, const void* bits, uint32_t bits_stride, const void* source_epoch,
                                const void* target_epoch, const void* data_root32, uint32_t n_agg, const void* att_status_out, const void* kind_out,
                                const void* n_flagged_out) {
    REQUIRE(ctx && members && off && bits && source_epoch && target_epoch && data_root32 && att_status_out && kind_out && n_flagged_out && n_agg > 0 &&
                bits_stride > 0,
            "slasher_update: bad arguments");
    return ctx->sl.H ? B2_OK : reject(ctx, "slasher_update", "no slasher (b2_slasher_init)");
}
int b2_slasher_update_dev(b2_ctx* ctx, const uint32_t* d_members, const uint32_t* d_off, const uint8_t* d_bits, uint32_t bits_stride,
                          const uint64_t* d_source_epoch, const uint64_t* d_target_epoch, const uint8_t* d_data_root32, const uint8_t* d_accept,
                          uint32_t n_agg, int32_t* d_att_status_out, uint8_t* d_kind_out, uint32_t* d_conflict_target_out, uint32_t* d_n_flagged_out,
                          void* stream) {
    B2_NVTX;
    int rc;
    if ((rc = check_slasher_update(ctx, d_members, d_off, d_bits, bits_stride, d_source_epoch, d_target_epoch, d_data_root32, n_agg, d_att_status_out, d_kind_out,
                                   d_n_flagged_out)))
        return rc;
    CK(cudaSetDevice(ctx->device));
    cudaStream_t s = (cudaStream_t)stream;
    if ((rc = ensure(ctx, ctx->sl.agg_id, (size_t)n_agg * 4))) return rc;
    const slasher_view S = slasher_view_of(ctx->sl);
    uint32_t* ids = ctx->sl.agg_id;
    CK(cudaMemsetAsync(d_n_flagged_out, 0, 4, s));
    k_slasher_rows<<<blocks_for(n_agg, 128), 128, 0, s>>>(S, d_off, bits_stride, d_source_epoch, d_target_epoch, d_data_root32, d_accept, n_agg,
                                                          d_att_status_out, ids, ctx->d_guard);
    CKL(ctx);
    k_slasher_record<<<n_agg, 128, 0, s>>>(S, d_members, d_off, d_bits, bits_stride, d_source_epoch, d_target_epoch, ids, n_agg, ctx->d_guard);
    CKL(ctx);
    k_slasher_check<<<n_agg, 128, 0, s>>>(S, d_members, d_off, d_bits, bits_stride, d_source_epoch, d_target_epoch, ids, n_agg, d_kind_out,
                                          d_conflict_target_out, d_n_flagged_out);
    CKL(ctx);
    return B2_OK;
}

int b2_slasher_update(b2_ctx* ctx, const uint32_t* members, const uint32_t* off, const uint8_t* bits, uint32_t bits_stride,
                      const uint64_t* source_epoch, const uint64_t* target_epoch, const uint8_t* data_root32, const uint8_t* accept, uint32_t n_agg,
                      int32_t* att_status_out, uint8_t* kind_out, uint32_t* conflict_target_out, uint32_t* n_flagged_out) {
    B2_NVTX;
    int rc;
    if ((rc = check_slasher_update(ctx, members, off, bits, bits_stride, source_epoch, target_epoch, data_root32, n_agg, att_status_out, kind_out, n_flagged_out)) ||
        (rc = check_batch(ctx, members, off, bits_stride, n_agg, ctx->sl.n_val, "slasher_update")))
        return rc;
    for (uint32_t a = 0; a < n_agg; a++)
        REQUIRE(source_epoch[a] < 0xffffffffull && target_epoch[a] < 0xffffffffull, "slasher_update: epoch does not fit 32 bits");
    CK(cudaSetDevice(ctx->device));
    staging st(ctx);
    const size_t total = off[n_agg];
    const uint32_t* dm = st.in(members, total, 4);
    const uint32_t* dof = st.in(off, (size_t)n_agg + 1);
    const uint8_t* db = st.in(bits, (size_t)n_agg * bits_stride, 16);
    const uint64_t* dse = st.in(source_epoch, n_agg);
    const uint64_t* dte = st.in(target_epoch, n_agg);
    const uint8_t* droot = st.in(data_root32, (size_t)n_agg * 32);
    const uint8_t* dacc = accept ? st.in(accept, n_agg) : nullptr;
    int32_t* dst = st.out(att_status_out, n_agg);
    uint8_t* dkind = st.out(kind_out, total);
    uint32_t* dconf = conflict_target_out ? st.out(conflict_target_out, 2 * total) : nullptr;
    uint32_t* dflag = st.out(n_flagged_out, 1);
    if ((rc = st.rc) ||
        (rc = b2_slasher_update_dev(ctx, dm, dof, db, bits_stride, dse, dte, droot, dacc, n_agg, dst, dkind, dconf, dflag, ctx->s_main)))
        return rc;
    return st.finish();
}

// ------------------------------------------------------------------------------------------ equivocation discounting (:1405-1461)
static int check_slasher_discount(b2_ctx* ctx, const void* members, const void* kind, uint64_t n_slots, const void* new_out, const void* n_new_out) {
    REQUIRE(ctx && members && kind && new_out && n_new_out && n_slots > 0 && n_slots < (1ull << 32), "slasher_discount: bad arguments");
    REQUIRE(ctx->n_val > 0, "slasher_discount: registry not loaded");
    return ctx->sl.H ? B2_OK : reject(ctx, "slasher_discount", "no slasher (b2_slasher_init)");
}
int b2_slasher_discount_dev(b2_ctx* ctx, const uint32_t* d_members, const uint8_t* d_kind, uint64_t n_slots, uint8_t* d_new_out,
                            uint32_t* d_n_new_out, void* stream) {
    B2_NVTX;
    int rc;
    if ((rc = check_slasher_discount(ctx, d_members, d_kind, n_slots, d_new_out, d_n_new_out))) return rc;
    CK(cudaSetDevice(ctx->device));
    cudaStream_t s = (cudaStream_t)stream;
    const slasher_tables& t = ctx->sl;
    CK(cudaMemsetAsync(d_n_new_out, 0, 4, s));
    k_slasher_discount<<<blocks_for(n_slots, 256), 256, 0, s>>>(d_members, d_kind, n_slots, ctx->n_val, t.v_begin, t.n_rows, ctx->reg.equiv,
                                                                d_new_out, d_n_new_out);
    CKL(ctx);
    CK(cudaEventRecord(ctx->ev_equiv_done, s));      // the next epoch tail's LMD update waits for it
    return B2_OK;
}

int b2_slasher_discount(b2_ctx* ctx, const uint32_t* members, const uint8_t* kind, uint64_t n_slots, uint8_t* new_out, uint32_t* n_new_out) {
    B2_NVTX;
    int rc;
    if ((rc = check_slasher_discount(ctx, members, kind, n_slots, new_out, n_new_out))) return rc;
    CK(cudaSetDevice(ctx->device));
    staging st(ctx);
    const uint32_t* dm = st.in(members, n_slots);
    const uint8_t* dk = st.in(kind, n_slots);
    uint8_t* dnew = st.out(new_out, n_slots);
    uint32_t* dn = st.out(n_new_out, 1);
    if ((rc = st.rc) || (rc = b2_slasher_discount_dev(ctx, dm, dk, n_slots, dnew, dn, ctx->s_main))) return rc;
    return st.finish();
}

int b2_equivocating_read(b2_ctx* ctx, uint8_t* out, uint64_t n_validators) {
    B2_NVTX;
    REQUIRE(ctx && out && n_validators == ctx->n_val && n_validators > 0, "equivocating_read: bad arguments / registry size");
    CK(cudaSetDevice(ctx->device));
    CK(cudaStreamWaitEvent(ctx->s_main, ctx->ev_equiv_done, 0));      // the marks enqueued on other streams so far
    staging st(ctx);
    st.out(out, ctx->reg.equiv, n_validators);
    return st.finish();
}

int b2_equivocating_slice_dev(b2_ctx* ctx, uint64_t v_begin, uint64_t v_end, uint8_t* d_out, void* stream) {
    B2_NVTX;
    REQUIRE(ctx && d_out && v_begin < v_end && v_end <= ctx->n_val, "equivocating_slice_dev: bad arguments / registry not loaded");
    CK(cudaSetDevice(ctx->device));
    CK(cudaMemcpyAsync(d_out, (const uint8_t*)ctx->reg.equiv + v_begin, v_end - v_begin, cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
    return B2_OK;
}

int b2_equivocating_merge_dev(b2_ctx* ctx, uint64_t v_begin, uint64_t v_end, const uint8_t* d_table, void* stream) {
    B2_NVTX;
    REQUIRE(ctx && d_table && v_begin < v_end && v_end <= ctx->n_val, "equivocating_merge_dev: bad arguments / registry not loaded");
    CK(cudaSetDevice(ctx->device));
    cudaStream_t s = (cudaStream_t)stream;
    k_equiv_merge<<<blocks_for(v_end - v_begin, 256), 256, 0, s>>>(d_table, v_begin, v_end - v_begin, ctx->reg.equiv);
    CKL(ctx);
    CK(cudaEventRecord(ctx->ev_equiv_done, s));
    return B2_OK;
}

// ------------------------------------------------------------------------------------------ block packing (pack.cuh)
static int check_pack_attestations(b2_ctx* ctx, const void* members, const void* committee_off, const void* committee_table, uint32_t n_committees,
                                   const void* cand_committee, const void* cand_data, const void* cand_flag_mask, const void* bits, uint32_t bits_stride,
                                   const void* sig96, uint32_t n_cand, uint32_t max_out, uint64_t effective_balance_increment, const void* n_out,
                                   const void* out_committee, const void* out_data, const void* out_bits, const void* out_sig96, const void* out_numerator,
                                   const void* out_src_off, const void* out_src, const void* cand_status) {
    REQUIRE(ctx && committee_off && (n_committees == 0 || (members && committee_table)) &&
                (n_cand == 0 || (cand_committee && cand_data && cand_flag_mask && bits && sig96 && out_src && cand_status)) && n_out && out_committee &&
                out_data && out_bits && out_sig96 && out_numerator && out_src_off && max_out > 0 && bits_stride > 0 && bits_stride <= PACK_MAX_WORDS * 4 &&
                effective_balance_increment > 0,
            "pack_attestations: bad arguments (max_out > 0, 0 < bits_stride <= 256, increment > 0)");
    return ctx->n_val > 0 ? B2_OK : reject(ctx, "pack_attestations", "registry not loaded");
}
int b2_pack_attestations_dev(b2_ctx* ctx, const uint32_t* d_members, const uint32_t* d_committee_off, const uint8_t* d_committee_table,
                             uint32_t n_committees, const uint32_t* d_cand_committee, const uint32_t* d_cand_data, const uint8_t* d_cand_flag_mask,
                             const uint8_t* d_bits, uint32_t bits_stride, const uint8_t* d_sig96, uint32_t n_cand, uint32_t max_out,
                             uint64_t effective_balance_increment, uint64_t base_reward_per_increment, uint32_t* d_n_out, uint32_t* d_out_committee,
                             uint32_t* d_out_data, uint8_t* d_out_bits, uint8_t* d_out_sig96, uint64_t* d_out_numerator, uint32_t* d_out_src_off,
                             uint32_t* d_out_src, uint8_t* d_cand_status, void* stream) {
    B2_NVTX;
    int rc;
    if ((rc = check_pack_attestations(ctx, d_members, d_committee_off, d_committee_table, n_committees, d_cand_committee, d_cand_data, d_cand_flag_mask, d_bits,
                                      bits_stride, d_sig96, n_cand, max_out, effective_balance_increment, d_n_out, d_out_committee, d_out_data, d_out_bits,
                                      d_out_sig96, d_out_numerator, d_out_src_off, d_out_src, d_cand_status)))
        return rc;
    CK(cudaSetDevice(ctx->device));
    cudaStream_t s = (cudaStream_t)stream;
    const size_t C = std::max<uint32_t>(n_cand, 1), K = n_committees, M = max_out, wstride = (bits_stride + 3) / 4;
    const size_t claim_words = 2 * ((ctx->n_val + 31) / 32);
    const registry_tables& R = ctx->reg;
    pack_view P = {};
    P.members = d_members;
    P.coff = d_committee_off;
    P.ctable = d_committee_table;
    P.cand_comm = d_cand_committee;
    P.cand_data = d_cand_data;
    P.cand_mask = d_cand_flag_mask;
    P.bits = d_bits;
    P.eff = R.eff;
    P.part[0] = R.part[0];
    P.part[1] = R.part[1];
    P.n_comm = n_committees;
    P.n_cand = n_cand;
    P.stride = bits_stride;
    P.wstride = (uint32_t)wstride;
    P.max_out = max_out;
    P.n_val = ctx->n_val;
    P.inc = effective_balance_increment;
    P.per_inc = base_reward_per_increment;
    P.cand_status = d_cand_status;
    P.guard = ctx->d_guard;
    // the decompressed candidate signatures (read by the kernels through P.dec_st), the gathered constituents and their segment sums
    uint8_t *st, *gst;
    uint32_t *aff, *gaff, *sumjac;
    int32_t* segst;
    scratch sc(ctx, ctx->pk);
    sc(P.cnt, K); sc(P.off, K + 1); sc(P.list, C); sc(P.fold_of, C); sc(P.fdata, C); sc(P.fcnt, C); sc(P.frow, C * wstride); sc(P.fmask, C);
    sc(P.egain, C); sc(P.eslot, C); sc(P.claim, claim_words); sc(P.dcomm, C); sc(P.dmask, C); sc(P.ctl, 4); sc(P.sel, M); sc(P.ord, M);
    sc(aff, C * 48, 16); sc(st, C, 16); sc(gaff, C * 48, 16); sc(gst, C, 16); sc(sumjac, M * 72); sc(segst, M);
    if (sc.rc) return sc.rc;
    P.dec_st = st;
    CK(cudaMemsetAsync(P.ctl, 0, 16, s));
    CK(cudaMemsetAsync(P.claim, 0, claim_words * 4, s));
    if (K) CK(cudaMemsetAsync(P.cnt, 0, K * 4, s));
    if (n_cand) {
        CK(cudaMemsetAsync(P.dcomm, 0xff, (size_t)n_cand * 4, s));
        CK(cudaMemsetAsync(P.dmask, 0xff, (size_t)n_cand * 4, s));
        CK(cudaMemsetAsync(d_out_src, 0, (size_t)n_cand * 4, s));
        k_g2_decompress<<<blocks_for(n_cand, ctx->dec_block), ctx->dec_block, 0, s>>>(d_sig96, n_cand, aff, st);
        CKL(ctx);
    }
    if (K) {
        k_pack_claim<<<n_committees, 128, 0, s>>>(P);
        CKL(ctx);
    }
    if (n_cand) {
        k_pack_prep<<<blocks_for(n_cand, 128), 128, 0, s>>>(P);
        CKL(ctx);
    }
    k_pack_scan<<<1, 1024, 0, s>>>(P);
    CKL(ctx);
    if (n_cand) {
        k_pack_scatter<<<blocks_for(n_cand, 128), 128, 0, s>>>(P);
        CKL(ctx);
    }
    if (K) {
        k_pack_committee<<<n_committees, 256, PACK_SMEM_ROWS, s>>>(P);
        CKL(ctx);
    }
    k_pack_select<<<1, 1024, 0, s>>>(P);
    CKL(ctx);
    k_pack_rank<<<blocks_for(max_out, 128), 128, 0, s>>>(P);
    CKL(ctx);
    k_pack_offsets<<<1, 1024, 0, s>>>(P, d_out_src_off, d_n_out);
    CKL(ctx);
    k_pack_emit<<<max_out, 128, 0, s>>>(P, d_out_src_off, d_out_committee, d_out_data, d_out_bits, (unsigned long long*)d_out_numerator, d_out_src);
    CKL(ctx);
    if (n_cand) {
        k_pack_gather<<<blocks_for(n_cand, 128), 128, 0, s>>>(aff, st, d_out_src, d_out_src_off + max_out, gaff, gst);
        CKL(ctx);
    }
    k_g2_segment_sum<<<max_out, 32, 0, s>>>(gaff, gst, d_out_src_off, max_out, sumjac, segst, n_cand, ctx->d_guard);
    CKL(ctx);
    k_g2_finish<<<blocks_for(max_out, 32), 32, 0, s>>>(sumjac, segst, max_out, d_out_sig96, nullptr, nullptr);
    CKL(ctx);
    if (n_cand) {
        k_pack_single<<<blocks_for(max_out, 128), 128, 0, s>>>(d_sig96, d_out_src_off, d_out_src, max_out, d_out_sig96);
        CKL(ctx);
    }
    return B2_OK;
}

int b2_pack_attestations(b2_ctx* ctx, const uint32_t* members, const uint32_t* committee_off, const uint8_t* committee_table, uint32_t n_committees,
                         const uint32_t* cand_committee, const uint32_t* cand_data, const uint8_t* cand_flag_mask, const uint8_t* bits, uint32_t bits_stride,
                         const uint8_t* sig96, uint32_t n_cand, uint32_t max_out, uint64_t effective_balance_increment, uint64_t base_reward_per_increment,
                         uint32_t* n_out, uint32_t* out_committee, uint32_t* out_data, uint8_t* out_bits, uint8_t* out_sig96, uint64_t* out_numerator,
                         uint32_t* out_src_off, uint32_t* out_src, uint8_t* cand_status) {
    B2_NVTX;
    int rc;
    if ((rc = check_pack_attestations(ctx, members, committee_off, committee_table, n_committees, cand_committee, cand_data, cand_flag_mask, bits, bits_stride, sig96,
                                      n_cand, max_out, effective_balance_increment, n_out, out_committee, out_data, out_bits, out_sig96, out_numerator,
                                      out_src_off, out_src, cand_status)) ||
        (rc = check_batch(ctx, members, committee_off, bits_stride, n_committees, ctx->n_val, "pack_attestations")))
        return rc;
    // the committees of one table are pairwise disjoint and repeat no member
    std::vector<uint8_t> claimed(2 * ctx->n_val, 0);
    for (uint32_t k = 0; k < n_committees; k++) {
        REQUIRE(committee_table[k] <= 1, "pack_attestations: committee_table entries are 0 (current) or 1 (previous)");
        uint8_t* seen = claimed.data() + (size_t)committee_table[k] * ctx->n_val;
        for (uint32_t i = committee_off[k]; i < committee_off[k + 1]; i++) {
            REQUIRE(!seen[members[i]], "pack_attestations: committees of one participation table overlap or repeat a member");
            seen[members[i]] = 1;
        }
    }
    // one data id = one AttestationData: one committee and one flag mask
    std::vector<uint32_t> dcomm(n_cand, PACK_NONE), dmask(n_cand, PACK_NONE);
    for (uint32_t c = 0; c < n_cand; c++) {
        REQUIRE(cand_committee[c] < n_committees, "pack_attestations: candidate committee index out of range");
        REQUIRE(cand_data[c] < n_cand, "pack_attestations: data id >= n_cand");
        const uint32_t d = cand_data[c], m = cand_flag_mask[c] & 7u;
        REQUIRE((dcomm[d] == PACK_NONE || dcomm[d] == cand_committee[c]) && (dmask[d] == PACK_NONE || dmask[d] == m),
                "pack_attestations: a data id with two committees or two flag masks");
        dcomm[d] = cand_committee[c];
        dmask[d] = m;
    }
    CK(cudaSetDevice(ctx->device));
    staging st(ctx);
    const uint32_t* dm = st.in(members, n_committees ? committee_off[n_committees] : 0, 4);
    const uint32_t* doff = st.in(committee_off, (size_t)n_committees + 1);
    const uint8_t* dtab = st.in(committee_table, n_committees, 4);
    const uint32_t* dcc = st.in(cand_committee, n_cand, 4);
    const uint32_t* dcd = st.in(cand_data, n_cand, 4);
    const uint8_t* dcm = st.in(cand_flag_mask, n_cand, 4);
    const uint8_t* db = st.in(bits, (size_t)n_cand * bits_stride, 16);
    const uint8_t* dsig = st.in(sig96, (size_t)n_cand * 96, 16);
    uint32_t* dn = st.out(n_out, 1);
    uint32_t* dk = st.out(out_committee, max_out);
    uint32_t* dd = st.out(out_data, max_out);
    uint8_t* dbits = st.out(out_bits, (size_t)max_out * bits_stride);
    uint8_t* dsig96 = st.out(out_sig96, (size_t)max_out * 96);
    uint64_t* dnum = st.out(out_numerator, max_out);
    uint32_t* dsoff = st.out(out_src_off, (size_t)max_out + 1);
    uint32_t* dsrc = n_cand ? st.out(out_src, n_cand) : nullptr;
    uint8_t* dstat = n_cand ? st.out(cand_status, n_cand) : nullptr;
    if ((rc = st.rc) || (rc = b2_pack_attestations_dev(ctx, dm, doff, dtab, n_committees, dcc, dcd, dcm, db, bits_stride, dsig, n_cand, max_out,
                                                       effective_balance_increment, base_reward_per_increment, dn, dk, dd, dbits, dsig96, dnum, dsoff, dsrc,
                                                       dstat, ctx->s_main)))
        return rc;
    return st.finish();
}

// ------------------------------------------------------------------------------------------ block tree
int b2_tree_load(b2_ctx* ctx, const uint32_t* parent, const uint64_t* slot, const uint8_t* root32, const uint8_t* leaf_viable, uint32_t n) {
    B2_NVTX;
    REQUIRE(ctx && parent && slot && root32 && leaf_viable && n > 0, "tree_load: bad arguments");
    for (uint32_t b = 1; b < n; b++) REQUIRE(parent[b] < b, "tree_load: blocks must be in topological order (parent[b] < b)");
    // children in CSR form
    std::vector<uint32_t> child_off(n + 1, 0), child_idx(n > 1 ? n - 1 : 0), fill(n, 0);
    for (uint32_t b = 1; b < n; b++) child_off[parent[b] + 1]++;
    for (uint32_t b = 0; b < n; b++) child_off[b + 1] += child_off[b];
    for (uint32_t b = 1; b < n; b++) child_idx[child_off[parent[b]] + fill[parent[b]]++] = b;
    // DFS pre-order numbering and subtree sizes
    std::vector<uint32_t> pre(n), size(n, 1), stack;
    stack.reserve(n);
    stack.push_back(0);
    uint32_t counter = 0;
    while (!stack.empty()) {
        uint32_t b = stack.back();
        stack.pop_back();
        pre[b] = counter++;
        for (uint32_t k = child_off[b + 1]; k > child_off[b]; k--) stack.push_back(child_idx[k - 1]);
    }
    for (uint32_t b = n - 1; b >= 1; b--) size[parent[b]] += size[b];
    // get_filtered_block_tree: keep a block iff a viable leaf lies below it
    std::vector<uint8_t> keep(n, 0);
    for (uint32_t b = 0; b < n; b++)
        if (child_off[b + 1] == child_off[b]) keep[b] = leaf_viable[b] ? 1 : 0;
    for (uint32_t b = n - 1; b >= 1; b--)
        if (keep[b]) keep[parent[b]] = 1;
    // lexicographic rank of the roots (the tie-break of get_head compares 32-byte roots)
    std::vector<uint32_t> order(n), rank(n);
    for (uint32_t b = 0; b < n; b++) order[b] = b;
    std::sort(order.begin(), order.end(), [&](uint32_t x, uint32_t y) {
        int c = memcmp(root32 + 32ull * x, root32 + 32ull * y, 32);
        return c != 0 ? c < 0 : x < y;
    });
    for (uint32_t i = 0; i < n; i++) rank[order[i]] = i;
    CK(cudaSetDevice(ctx->device));
    int rc;
    // the new form and tables replace the old ones only once complete, so a failed load leaves the tree as it was
    tree_tables t;
    t.form = tree_form_of(n);
    const bool smem = t.form.smem_tree;
    // the tables of the tree's form, in pre-order.  A shared-memory tree has at most 15 * 1024 blocks: size and rank fit 15 bits.
    std::vector<uint32_t> inv(n), packed(smem ? n : 0), size_keep(smem ? 0 : n), rank_p(smem ? 0 : n);
    for (uint32_t b = 0; b < n; b++) {
        const uint32_t p = pre[b], k = keep[b] ? 0x80000000u : 0u;
        inv[p] = b;
        if (smem) {
            packed[p] = size[b] | (rank[b] << 15) | k;
        } else {
            size_keep[p] = size[b] | k;
            rank_p[p] = rank[b];
        }
    }
    const size_t n4 = (size_t)n * 4, n8 = (size_t)n * 8;
    if ((rc = ensure(ctx, t.pre, n4)) || (rc = ensure(ctx, t.inv, n4)) || (rc = ensure(ctx, t.head, 4)) || (rc = ensure(ctx, t.votes, n8)) ||
        (rc = ensure(ctx, t.weight, n8)))
        return rc;
    if (smem && (rc = ensure(ctx, t.packed, n4))) return rc;
    if (!smem && ((rc = ensure(ctx, t.size_keep, n4)) || (rc = ensure(ctx, t.rank, n4)) || (rc = ensure(ctx, t.next, n4 + 4)) ||
                  (rc = ensure(ctx, t.prefix, n8 + 8)) || (rc = ensure(ctx, t.w2, n8))))
        return rc;
    if ((rc = ensure(ctx, t.size, n4)) || (rc = ensure(ctx, t.rank_id, n4)) || (rc = ensure(ctx, t.parent, n4)) || (rc = ensure(ctx, t.root, 32ull * n)) ||
        (rc = ensure(ctx, t.viable, n)) || (rc = ensure(ctx, t.slot, n8)))
        return rc;
    cudaStream_t s = ctx->s_main;
    CK(cudaMemcpyAsync(t.size, size.data(), n4, cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync(t.rank_id, rank.data(), n4, cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync(t.parent, parent, n4, cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync(t.root, root32, 32ull * n, cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync(t.viable, leaf_viable, n, cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync(t.slot, slot, n8, cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync(t.pre, pre.data(), n4, cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync(t.inv, inv.data(), n4, cudaMemcpyHostToDevice, s));
    if (smem) {
        CK(cudaMemcpyAsync(t.packed, packed.data(), n4, cudaMemcpyHostToDevice, s));
    } else {
        CK(cudaMemcpyAsync(t.size_keep, size_keep.data(), n4, cudaMemcpyHostToDevice, s));
        CK(cudaMemcpyAsync(t.rank, rank_p.data(), n4, cudaMemcpyHostToDevice, s));
    }
    CK(cudaMemsetAsync(t.votes, 0, n8, s));
    CK(cudaStreamSynchronize(s));
    ctx->tree = std::move(t);
    ctx->n_blocks = n;
    return B2_OK;
}

// Room for a change from n_old blocks to n, all or nothing: every buffer too small for it is first allocated anew (geometrically, so
// one block per slot does not reallocate each time) with the live contents copied over -- the per-id state and the tables of the current
// form keep their n_old entries -- and only once every allocation has succeeded do the new buffers replace the old ones.  A failed
// allocation therefore leaves the tree exactly as it was.  The scratch holds max(n_old, n) entries; the tables of n's form are
// re-emitted after the change.
static int tree_reserve(b2_ctx* ctx, uint32_t n_old, uint32_t n) {
    tree_tables& t = ctx->tree;
    const size_t k4 = (size_t)n_old * 4, m = std::max(n_old, n), m4 = m * 4, n4 = (size_t)n * 4, n8 = (size_t)n * 8;
    const bool smem = tree_form_of(n).smem_tree;
    struct want {
        dbuf* b;
        size_t keep, need;
    };
    const want all[] = {{&t.pre, k4, m4}, {&t.size, k4, m4}, {&t.rank_id, k4, m4}, {&t.parent, k4, m4}, {&t.root, 32 * (size_t)n_old, 32 * m},
                        {&t.viable, n_old, m}, {&t.slot, 8 * (size_t)n_old, 8 * m}, {&t.pre_b, 0, m4}, {&t.size_b, 0, m4}, {&t.rank_b, 0, m4},
                        {&t.parent_b, 0, m4}, {&t.root_b, 0, 32 * m}, {&t.viable_b, 0, m}, {&t.slot_b, 0, 8 * m}, {&t.scan, 0, m4 + 4}, {&t.scan2, 0, m4 + 4}, {&t.map, 0, m4},
                        {&t.inv, k4, n4}, {&t.votes, 8 * (size_t)std::min(n_old, n), n8}, {&t.weight, 0, n8},
                        {&t.packed, k4, smem ? n4 : 0}, {&t.size_keep, k4, smem ? 0 : n4}, {&t.rank, k4, smem ? 0 : n4},
                        {&t.next, 0, smem ? 0 : n4 + 4}, {&t.prefix, 0, smem ? 0 : n8 + 8}, {&t.w2, 0, smem ? 0 : n8}};
    constexpr size_t N_BUF = sizeof(all) / sizeof(all[0]);
    dbuf fresh[N_BUF];
    for (size_t i = 0; i < N_BUF; i++) {
        const dbuf& b = *all[i].b;
        if (!all[i].need || (b.p && all[i].need <= b.cap)) continue;
        const size_t bytes = std::max<size_t>({all[i].need, 2 * b.cap, 256}), keep = b.p ? std::min(all[i].keep, b.cap) : 0;
        CK(cudaMalloc(&fresh[i].p, bytes));
        fresh[i].cap = bytes;
        if (keep) CK(cudaMemcpyAsync(fresh[i].p, b.p, keep, cudaMemcpyDeviceToDevice, ctx->s_main));
    }
    for (size_t i = 0; i < N_BUF; i++)
        if (fresh[i]) *all[i].b = std::move(fresh[i]);
    return B2_OK;
}

static tree_ids ids_of(tree_tables& t, bool other) {
    return other ? tree_ids{t.pre_b, t.size_b, t.rank_b, t.parent_b, t.root_b, t.viable_b, t.slot_b}
                 : tree_ids{t.pre, t.size, t.rank_id, t.parent, t.root, t.viable, t.slot};
}

// re-emits the tables of the form of an n-block tree, waits for the change, and makes n the tree's size
static int tree_emit(b2_ctx* ctx, uint32_t n) {
    tree_tables& t = ctx->tree;
    const tree_form f = tree_form_of(n);
    k_tree_emit<<<1, 1024, 0, ctx->s_main>>>(t.pre, t.size, t.rank_id, t.viable, n, t.scan, t.inv, f.smem_tree ? (uint32_t*)t.packed : nullptr,
                                             t.size_keep, t.rank);
    CKL(ctx);
    CK(cudaStreamSynchronize(ctx->s_main));
    t.form = f;
    ctx->n_blocks = n;
    return B2_OK;
}

int b2_tree_add(b2_ctx* ctx, const uint32_t* parent, const uint64_t* slot, const uint8_t* root32, const uint8_t* leaf_viable, uint32_t k) {
    B2_NVTX;
    REQUIRE(ctx && parent && slot && root32 && leaf_viable, "tree_add: bad arguments");
    REQUIRE(ctx->n_blocks > 0, "tree_add: no tree loaded (b2_tree_load)");
    const uint32_t n0 = ctx->n_blocks;
    REQUIRE(k > 0 && k < 0xffffffffu - n0, "tree_add: k must be at least 1 and the tree below 2^32 - 1 blocks");
    for (uint32_t j = 0; j < k; j++) REQUIRE(parent[j] < n0 + j, "tree_add: a block's parent must precede it (parent < id)");
    CK(cudaSetDevice(ctx->device));
    const uint32_t n = n0 + k;
    int rc;
    if ((rc = tree_reserve(ctx, n0, n))) return rc;
    tree_tables& t = ctx->tree;
    cudaStream_t s = ctx->s_main;
    // the new blocks' inputs go past the current n, where nothing reads them until the change is complete
    CK(cudaMemcpyAsync((uint32_t*)t.parent + n0, parent, (size_t)k * 4, cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync((uint8_t*)t.root + 32ull * n0, root32, 32ull * k, cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync((uint8_t*)t.viable + n0, leaf_viable, k, cudaMemcpyHostToDevice, s));
    CK(cudaMemcpyAsync((uint64_t*)t.slot + n0, slot, (size_t)k * 8, cudaMemcpyHostToDevice, s));
    CK(cudaMemsetAsync((uint64_t*)t.votes + n0, 0, (size_t)k * 8, s));      // the vote accumulator is clean between calls
    if (tree_form_of(n).smem_tree) {
        k_tree_insert_cta<<<1, 1024, 0, s>>>(t.pre, t.size, t.parent, n0, k);
        CKL(ctx);
    } else {
        for (uint32_t j = 0; j < k; j++) {
            k_tree_insert_grid<<<blocks_for(n0 + j + 1, 256), 256, 0, s>>>(t.pre, t.size, t.size_b, parent[j], n0 + j);
            CKL(ctx);
            std::swap(t.size, t.size_b);
        }
    }
    k_tree_rank_old<<<blocks_for(n0, 256), 256, 0, s>>>(t.root, t.rank_id, n0, n);
    CKL(ctx);
    k_tree_rank_new<<<k, 256, 0, s>>>(t.root, t.rank_id, n0, n);
    CKL(ctx);
    return tree_emit(ctx, n);
}

int b2_tree_prune(b2_ctx* ctx, uint32_t new_root, uint32_t* map_out) {
    B2_NVTX;
    REQUIRE(ctx && map_out, "tree_prune: bad arguments");
    REQUIRE(ctx->n_blocks > 0, "tree_prune: no tree loaded (b2_tree_load)");
    const uint32_t n0 = ctx->n_blocks;
    REQUIRE(new_root < n0, "tree_prune: new root out of range");
    CK(cudaSetDevice(ctx->device));
    tree_tables& t = ctx->tree;
    uint32_t n = 0;      // the kept subtree's size decides the new form, so it is read before anything is allocated
    CK(cudaMemcpy(&n, (uint32_t*)t.size + new_root, 4, cudaMemcpyDeviceToHost));
    int rc;
    if ((rc = tree_reserve(ctx, n0, n))) return rc;
    cudaStream_t s = ctx->s_main;
    k_tree_prune<<<1, 1024, 0, s>>>(ids_of(t, false), ids_of(t, true), n0, new_root, t.scan, t.scan2, t.map);
    CKL(ctx);
    if (ctx->n_val > 0) {
        k_lmd_remap<<<blocks_for(ctx->n_val, 256), 256, 0, s>>>(ctx->reg.lmd_block, ctx->n_val, t.map, n0);
        CKL(ctx);
    }
    std::swap(t.pre, t.pre_b), std::swap(t.size, t.size_b), std::swap(t.rank_id, t.rank_b);
    std::swap(t.parent, t.parent_b), std::swap(t.root, t.root_b), std::swap(t.viable, t.viable_b), std::swap(t.slot, t.slot_b);
    CK(cudaMemcpyAsync(map_out, t.map, (size_t)n0 * 4, cudaMemcpyDeviceToHost, s));
    return tree_emit(ctx, n);
}

int b2_tree_set_viable(b2_ctx* ctx, const uint32_t* idx, const uint8_t* viable, uint32_t k) {
    B2_NVTX;
    REQUIRE(ctx && idx && viable, "tree_set_viable: bad arguments");
    REQUIRE(ctx->n_blocks > 0, "tree_set_viable: no tree loaded (b2_tree_load)");
    REQUIRE(k > 0, "tree_set_viable: k must be at least 1");
    for (uint32_t j = 0; j < k; j++) REQUIRE(idx[j] < ctx->n_blocks, "tree_set_viable: block index out of range");
    CK(cudaSetDevice(ctx->device));
    const uint32_t n = ctx->n_blocks;
    int rc;
    if ((rc = tree_reserve(ctx, n, n))) return rc;
    staging st(ctx);
    const uint32_t* didx = st.in(idx, k);
    const uint8_t* dval = st.in(viable, k);
    if (st.rc) return st.rc;
    k_tree_set_viable<<<1, 1, 0, ctx->s_main>>>(ctx->tree.viable, didx, dval, k);
    CKL(ctx);
    return tree_emit(ctx, n);
}

// the vote scatter's view of the validators [v_begin, v_end) under the context's fork-choice variant
static ghost_votes_args votes_args(const b2_ctx* ctx, uint64_t v_begin, uint64_t v_end) {
    const registry_tables& R = ctx->reg;
    return {v_end - v_begin, (unsigned long long*)R.lmd_key + v_begin, (uint32_t*)R.lmd_block + v_begin, (uint8_t*)R.equiv + v_begin,
            (uint8_t*)R.flags + v_begin, (uint64_t*)R.eff + v_begin, ctx->fc_min_key, 1u, ctx->fc_exclude_slashed ? 3u : 1u};
}

// the tree phase's (K9) view of the tree in its form, without host publication; it is launched with ctx->tree.form.tree_smem bytes of
// dynamic shared memory
static ghost_tree_args tree_args(const b2_ctx* ctx, uint64_t* d_votes_preorder, uint32_t justified_idx, int32_t boost_idx, uint64_t boost_score,
                                 uint64_t* d_weight_out, uint32_t* d_head_idx_out) {
    const tree_tables& T = ctx->tree;
    return {ctx->n_blocks, T.pre, T.inv, T.size_keep, T.rank, T.packed, (unsigned long long*)d_votes_preorder, T.prefix, T.w2, T.next,
            (unsigned long long*)d_weight_out, d_head_idx_out, nullptr, 0, justified_idx, boost_idx, boost_score, T.form.smem_tree,
            T.form.work_list, ctx->d_dbg};
}

// Spins on the mapped (head, sequence) slot until the get_head kernel on `s` has published call `seq`.  Every 2^20 polls it checks that
// the kernel is still alive; if it finished without publishing (should not happen), the head is copied from d_head instead.
static int wait_head(b2_ctx* ctx, uint32_t seq, cudaStream_t s, const char* what, uint32_t* head_idx_out) {
    volatile unsigned long long* slot64 = reinterpret_cast<volatile unsigned long long*>(ctx->h_head);
    unsigned long long got = 0;
    for (uint64_t spins = 0; (uint32_t)((got = *slot64) >> 32) != seq; spins++) {
        if ((spins & 0xfffff) == 0xfffff) {
            cudaError_t q = cudaStreamQuery(s);
            if (q != cudaErrorNotReady && q != cudaSuccess) return fail_cuda(ctx, q, what);
            if (q == cudaSuccess && (uint32_t)(*slot64 >> 32) != seq) {
                uint32_t h = 0;
                CK(cudaMemcpy(&h, ctx->tree.head, 4, cudaMemcpyDeviceToHost));
                *head_idx_out = h;
                return B2_OK;
            }
        }
    }
    *head_idx_out = (uint32_t)got;
    return B2_OK;
}

int b2_vote_weights_range_dev(b2_ctx* ctx, uint64_t v_begin, uint64_t v_end, uint64_t* d_votes_preorder, void* stream) {
    B2_NVTX;
    REQUIRE(ctx && d_votes_preorder, "vote_weights_dev: bad arguments");
    REQUIRE(ctx->n_val > 0 && ctx->n_blocks > 0, "vote_weights: registry or tree not loaded");
    REQUIRE(v_begin <= v_end && v_end <= ctx->n_val, "vote_weights_range: validator range outside the registry");
    CK(cudaSetDevice(ctx->device));
    cudaStream_t s = (cudaStream_t)stream;
    const ghost_votes_args V = votes_args(ctx, v_begin, v_end);
    const size_t bins_bytes = (size_t)ctx->n_blocks * 8;
    if (V.n > 0) {          // else nothing to scatter; the accumulator is clean by contract
        // the bins in shared memory when they fit (a persistent grid of at most one CTA per SM), else the global-atomic form
        const bool smem = ctx->tree.form.smem_bins;
        const unsigned grid = smem ? (unsigned)std::min<uint64_t>((uint64_t)ctx->n_sm, (V.n + 1023) / 1024) : blocks_for(V.n, 256);
        (smem ? k_ghost_votes_smem : k_ghost_votes)<<<grid, smem ? 1024 : 256, smem ? bins_bytes : 0, s>>>(
            V.n, V.lmd_key, V.lmd_block, V.equiv, V.flags, V.eff, ctx->tree.pre, ctx->n_blocks, (unsigned long long*)d_votes_preorder, V.min_key, V.flag_need,
            V.flag_mask);
        CKL(ctx);
    }
    CK(cudaEventRecord(ctx->ev_votes_done, s));
    return B2_OK;
}
int b2_vote_weights_dev(b2_ctx* ctx, uint64_t* d_votes_preorder, void* stream) {
    B2_NVTX;
    REQUIRE(ctx, "vote_weights_dev: bad arguments");
    return b2_vote_weights_range_dev(ctx, 0, ctx->n_val, d_votes_preorder, stream);
}

int b2_head_from_votes_dev(b2_ctx* ctx, uint64_t* d_votes_preorder, uint32_t justified_idx, int32_t boost_idx, uint64_t boost_score,
                           uint64_t* d_weight_out, uint32_t* d_head_idx_out, void* stream) {
    B2_NVTX;
    REQUIRE(ctx && d_votes_preorder && d_head_idx_out, "head_from_votes_dev: bad arguments");
    REQUIRE(ctx->n_blocks > 0, "head_from_votes: tree not loaded");
    REQUIRE(justified_idx < ctx->n_blocks && boost_idx < (int32_t)ctx->n_blocks, "head_from_votes: block index out of range");
    CK(cudaSetDevice(ctx->device));
    cudaStream_t s = (cudaStream_t)stream;
    k_ghost_tree<<<1, 1024, ctx->tree.form.tree_smem, s>>>(tree_args(ctx, d_votes_preorder, justified_idx, boost_idx, boost_score, d_weight_out, d_head_idx_out));
    CKL(ctx);
    return B2_OK;
}

int b2_get_weights(b2_ctx* ctx, int32_t boost_idx, uint64_t boost_score, uint64_t* weight_out) {
    B2_NVTX;
    REQUIRE(ctx && weight_out, "get_weights: bad arguments");
    REQUIRE(ctx->n_val > 0 && ctx->n_blocks > 0, "get_weights: registry or tree not loaded");
    int rc;
    cudaStream_t s = ctx->s_main;
    const tree_tables& T = ctx->tree;
    if ((rc = b2_vote_weights_dev(ctx, T.votes, s)) || (rc = b2_head_from_votes_dev(ctx, T.votes, 0, boost_idx, boost_score, T.weight, T.head, s))) return rc;
    staging st(ctx);
    st.out(weight_out, T.weight, ctx->n_blocks);
    return st.finish();
}

// ---- multi-GPU get_head with the all-reduce fused in over NVLink peer memory (k_get_head_fused_nvl)
static size_t fc_acc_bytes(uint32_t n_blocks) { return ((size_t)2 * n_blocks * 8 + 255) & ~(size_t)255; }
int b2_fc_exchange_export(b2_ctx* ctx, uint8_t* handle64_out) {
    B2_NVTX;
    REQUIRE(ctx && handle64_out, "fc_exchange_export: bad arguments");
    REQUIRE(ctx->n_blocks > 0, "fc_exchange_export: load the block tree first (the exchange block is sized by it)");
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle is 64 bytes");
    CK(cudaSetDevice(ctx->device));
    CK(cudaDeviceSynchronize());
    for (int r = 0; r < B2_MAX_PEERS; r++) {
        if (ctx->fc_peer[r] && r != ctx->fc_rank) CK(cudaIpcCloseMemHandle(ctx->fc_peer[r]));
        ctx->fc_peer[r] = nullptr;
    }
    ctx->fc_block = dbuf();
    ctx->fc_rank = -1;
    ctx->fc_world = 0;
    const size_t bytes = fc_acc_bytes(ctx->n_blocks) + 2 * B2_MAX_PEERS * sizeof(unsigned int);
    int rc;
    if ((rc = ensure(ctx, ctx->fc_block, bytes))) return rc;
    CK(cudaMemset(ctx->fc_block, 0, bytes));
    ctx->fc_blocks_cap = ctx->n_blocks;
    ctx->fc_seq = 0;
    cudaIpcMemHandle_t h;
    CK(cudaIpcGetMemHandle(&h, ctx->fc_block));
    memcpy(handle64_out, &h, 64);
    return B2_OK;
}
int b2_fc_exchange_open(b2_ctx* ctx, int rank, int world, const uint8_t* handles64) {
    B2_NVTX;
    REQUIRE(ctx && handles64 && world >= 1 && world <= B2_MAX_PEERS && rank >= 0 && rank < world, "fc_exchange_open: bad arguments");
    REQUIRE(ctx->fc_block, "fc_exchange_open: call b2_fc_exchange_export first");
    CK(cudaSetDevice(ctx->device));
    for (int r = 0; r < world; r++) {
        if (r == rank) {
            ctx->fc_peer[r] = ctx->fc_block;
            continue;
        }
        cudaIpcMemHandle_t h;
        memcpy(&h, handles64 + 64 * (size_t)r, 64);
        CK(cudaIpcOpenMemHandle(&ctx->fc_peer[r], h, cudaIpcMemLazyEnablePeerAccess));
    }
    ctx->fc_rank = rank;
    ctx->fc_world = world;
    return B2_OK;
}
int b2_get_head_multi(b2_ctx* ctx, uint64_t v_begin, uint64_t v_end, uint32_t justified_idx, int32_t boost_idx, uint64_t boost_score, uint32_t* head_idx_out) {
    B2_NVTX;
    REQUIRE(ctx && head_idx_out, "get_head_multi: bad arguments");
    REQUIRE(ctx->n_val > 0 && ctx->n_blocks > 0, "get_head_multi: registry or tree not loaded");
    REQUIRE(ctx->fc_world >= 1 && ctx->fc_blocks_cap == ctx->n_blocks, "get_head_multi: exchange block not opened for this tree (b2_fc_exchange_export / _open)");
    REQUIRE(v_begin <= v_end && v_end <= ctx->n_val, "get_head_multi: validator range outside the registry");
    REQUIRE(justified_idx < ctx->n_blocks && boost_idx < (int32_t)ctx->n_blocks, "get_head_multi: block index out of range");
    CK(cudaSetDevice(ctx->device));
    cudaStream_t s = ctx->s_main;
    REQUIRE(ctx->tree.form.smem_tree, "get_head_multi: the tree does not fit the shared-memory form (<= 14 463 blocks)");
    ghost_tree_args A = tree_args(ctx, ctx->tree.votes, justified_idx, boost_idx, boost_score, nullptr, ctx->tree.head);
    const ghost_votes_args V = votes_args(ctx, v_begin, v_end);
    ghost_peer_args P;
    const uint32_t seq = ++ctx->fc_seq ? ctx->fc_seq : ++ctx->fc_seq;                  // the collective call number (same on every rank)
    const uint32_t hseq = ++ctx->head_seq ? ctx->head_seq : ++ctx->head_seq;            // this context's host-slot sequence number
    for (int r = 0; r < B2_MAX_PEERS; r++) {
        P.acc[r] = r < ctx->fc_world ? (unsigned long long*)ctx->fc_peer[r] : nullptr;
        P.flags[r] = r < ctx->fc_world ? (unsigned int*)((char*)ctx->fc_peer[r] + fc_acc_bytes(ctx->n_blocks)) : nullptr;
    }
    P.rank = (uint32_t)ctx->fc_rank;
    P.world = (uint32_t)ctx->fc_world;
    P.seq = seq;
    A.host_out = ctx->d_head_host;
    A.host_seq = hseq;
    const unsigned grid = (unsigned)std::max<uint64_t>(1, std::min<uint64_t>((uint64_t)ctx->n_sm, (V.n + 1023) / 1024));
    k_get_head_fused_nvl<<<grid, 1024, ctx->tree.form.tree_smem, s>>>(V, A, P, ctx->d_ticket, ctx->tree.votes);
    CKL(ctx);
    CK(cudaEventRecord(ctx->ev_votes_done, s));
    return wait_head(ctx, hseq, s, "get_head_multi kernel", head_idx_out);
}

// Diagnostics: SM-clock stamps (clock64) of the phases of the LAST b2_get_head / b2_head_from_votes_dev of this context: out32[0..7] =
// tree phase boundaries (start, staged, scanned, weights, weights stored, marked, counted, head found), out32[15] = tree end,
// out32[16..19] = vote scatter of CTA 0 (start, bins zeroed, scattered, flushed).  For profiling (tools/), not for results.
// Only some forms write some slots (out32[3]: the shared-memory tree phase; out32[8]: its work-list marking; out32[16..19]: the one-launch
// kernels), so reading clears the stamps: a slot that no call since the last read has written reads 0.
int b2_debug_head_clocks(b2_ctx* ctx, uint64_t* out32) {
    REQUIRE(ctx && out32, "debug_head_clocks: bad arguments");
    CK(cudaSetDevice(ctx->device));
    CK(cudaDeviceSynchronize());
    staging st(ctx);
    uint64_t* d = st.out(out32, 32);
    if (st.rc) return st.rc;
    CK(cudaMemcpyAsync(d, ctx->d_dbg, 32 * 8, cudaMemcpyDeviceToDevice, ctx->s_main));
    CK(cudaMemsetAsync(ctx->d_dbg, 0, 32 * 8, ctx->s_main));
    return st.finish();
}

int b2_get_head(b2_ctx* ctx, uint32_t justified_idx, int32_t boost_idx, uint64_t boost_score, uint32_t* head_idx_out) {
    B2_NVTX;
    REQUIRE(ctx && head_idx_out, "get_head: bad arguments");
    REQUIRE(ctx->n_val > 0 && ctx->n_blocks > 0, "get_head: registry or tree not loaded");
    REQUIRE(justified_idx < ctx->n_blocks && boost_idx < (int32_t)ctx->n_blocks, "get_head: block index out of range");
    int rc;
    cudaStream_t s = ctx->s_main;
    if (ctx->head_fused && ctx->tree.form.smem_tree) {
        // one launch; the kernel writes (head, sequence) into mapped pinned memory and the host spins on the sequence number
        CK(cudaSetDevice(ctx->device));
        ghost_tree_args A = tree_args(ctx, ctx->tree.votes, justified_idx, boost_idx, boost_score, nullptr, ctx->tree.head);
        const ghost_votes_args V = votes_args(ctx, 0, ctx->n_val);
        const uint32_t seq = ++ctx->head_seq ? ctx->head_seq : ++ctx->head_seq;       // never 0
        A.host_out = ctx->d_head_host;
        A.host_seq = seq;
        const unsigned grid = (unsigned)std::min<uint64_t>((uint64_t)ctx->n_sm, (V.n + 1023) / 1024);
        k_get_head_fused<<<grid, 1024, ctx->tree.form.tree_smem, s>>>(V, A, ctx->d_ticket);
        CKL(ctx);
        CK(cudaEventRecord(ctx->ev_votes_done, s));
        return wait_head(ctx, seq, s, "get_head kernel", head_idx_out);
    }
    if ((rc = b2_vote_weights_dev(ctx, ctx->tree.votes, s))) return rc;
    if ((rc = b2_head_from_votes_dev(ctx, ctx->tree.votes, justified_idx, boost_idx, boost_score, nullptr, ctx->tree.head, s))) return rc;
    uint32_t h = 0;
    CK(cudaMemcpyAsync(&h, ctx->tree.head, 4, cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    *head_idx_out = h;
    return B2_OK;
}

// ------------------------------------------------------------------------------------------ hash_tree_root (ssz.cuh)
constexpr uint32_t SSZ_REGISTRY_DEPTH = 40;      // VALIDATOR_REGISTRY_LIMIT = 2^40

static const ssz_zero_hashes& ssz_zeros() {
    static const ssz_zero_hashes Z = [] {
        ssz_zero_hashes z = {};
        for (int l = 1; l < SSZ_MAX_DEPTH; l++) sha256_node_pair(z.z[l - 1], z.z[l - 1], z.z[l]);
        return z;
    }();
    return Z;
}

static uint32_t ssz_log2(uint64_t pow2) {
    uint32_t l = 0;
    while ((1ull << l) < pow2) l++;
    return l;
}

static uint64_t ssz_leaves_for(uint64_t n) {
    uint64_t C = 1;
    while (C < n) C <<= 1;
    return C;
}

// every inner node of a heap whose C leaves are in place: one subtree launch per SSZ_SUBTREE_LEVELS levels (2^20 leaves: 3 launches)
static int ssz_reduce(b2_ctx* ctx, uint32_t* cache, uint64_t C) {
    for (uint64_t m = C; m > 1;) {
        const uint32_t levels = std::min<uint32_t>(SSZ_SUBTREE_LEVELS, ssz_log2(m));
        k_ssz_subtree<<<(unsigned)(m >> levels), 256, 0, ctx->s_main>>>(cache, m, levels);
        CKL(ctx);
        m >>= levels;
    }
    return B2_OK;
}

// node 1 of the heap, padded with zero subtrees from depth log2 C to `depth`, then mixed with the length when mix_in is set
static int ssz_root(b2_ctx* ctx, const uint32_t* cache, uint64_t C, uint32_t depth, int mix_in, uint64_t length, uint8_t* d_root32) {
    k_ssz_root<<<1, 32, 0, ctx->s_main>>>(cache + 8, ssz_log2(C), depth, ssz_zeros(), mix_in, length, d_root32);
    CKL(ctx);
    return B2_OK;
}

int b2_ssz_validators_load(b2_ctx* ctx, const uint8_t* rec121, uint64_t n, uint8_t* root32_out) {
    B2_NVTX;
    REQUIRE(ctx && root32_out && (n == 0 || rec121) && n < (1ull << 32), "ssz_validators_load: bad arguments (n < 2^32)");
    CK(cudaSetDevice(ctx->device));
    ssz_tables t;      // built aside: a failed load leaves the previous cache answering
    t.n = n;
    t.C = ssz_leaves_for(n);
    int rc;
    if ((rc = ensure(ctx, t.cache, t.C * 64))) return rc;
    staging st(ctx);
    const uint8_t* drec = st.in(rec121, n * SSZ_VALIDATOR_BYTES);
    uint8_t* droot = st.out(root32_out, 32);
    if (st.rc) return st.rc;
    cudaStream_t s = ctx->s_main;
    if (n) {
        k_ssz_validator_leaves<<<blocks_for(n, SSZ_LEAF_THREADS), SSZ_LEAF_THREADS, 0, s>>>(drec, nullptr, n, t.cache, t.C);
        CKL(ctx);
    }
    CK(cudaMemsetAsync((uint32_t*)t.cache + (t.C + n) * 8, 0, (t.C - n) * 32, s));      // the zero leaves past n
    if ((rc = ssz_reduce(ctx, t.cache, t.C)) || (rc = ssz_root(ctx, t.cache, t.C, SSZ_REGISTRY_DEPTH, 1, n, droot)) || (rc = st.finish()))
        return rc;
    t.chunks = std::move(ctx->ssz.chunks);
    ctx->ssz = std::move(t);
    return B2_OK;
}

int b2_ssz_validators_update(b2_ctx* ctx, const uint32_t* idx, const uint8_t* rec121, uint64_t k, uint8_t* root32_out) {
    B2_NVTX;
    REQUIRE(ctx && root32_out && (k == 0 || (idx && rec121)), "ssz_validators_update: bad arguments");
    ssz_tables& t = ctx->ssz;
    REQUIRE(t.C, "ssz_validators_update: no validators tree (b2_ssz_validators_load)");
    for (uint64_t j = 0; j < k; j++)
        REQUIRE(idx[j] < t.n && (j == 0 || idx[j - 1] < idx[j]), "ssz_validators_update: indices must be strictly increasing and below n");
    CK(cudaSetDevice(ctx->device));
    staging st(ctx);
    const uint32_t* didx = st.in(idx, k);
    const uint8_t* drec = st.in(rec121, k * SSZ_VALIDATOR_BYTES);
    uint8_t* droot = st.out(root32_out, 32);
    if (st.rc) return st.rc;
    cudaStream_t s = ctx->s_main;
    if (k) {
        k_ssz_validator_leaves<<<blocks_for(k, SSZ_LEAF_THREADS), SSZ_LEAF_THREADS, 0, s>>>(drec, didx, k, t.cache, t.C);
        CKL(ctx);
        for (uint32_t shift = 1, depth = ssz_log2(t.C); shift <= depth; shift++) {
            k_ssz_update_level<<<blocks_for(k, 128), 128, 0, s>>>(t.cache, didx, k, t.C, shift);
            CKL(ctx);
        }
    }
    int rc;
    if ((rc = ssz_root(ctx, t.cache, t.C, SSZ_REGISTRY_DEPTH, 1, t.n, droot))) return rc;
    return st.finish();
}

int b2_ssz_chunks_root(b2_ctx* ctx, const uint8_t* data, uint64_t n_bytes, uint32_t limit_depth, int mix_in, uint64_t length,
                       uint8_t* root32_out) {
    B2_NVTX;
    REQUIRE(ctx && root32_out && (n_bytes == 0 || data) && n_bytes < (1ull << 40) && limit_depth <= SSZ_MAX_DEPTH,
            "ssz_chunks_root: bad arguments (n_bytes < 2^40, limit_depth <= 64)");
    const uint64_t C = ssz_leaves_for((n_bytes + 31) / 32);
    REQUIRE(ssz_log2(C) <= limit_depth, "ssz_chunks_root: more chunks than 2^limit_depth");
    CK(cudaSetDevice(ctx->device));
    int rc;
    if ((rc = ensure(ctx, ctx->ssz.chunks, C * 64))) return rc;
    staging st(ctx);
    const uint8_t* dd = st.in(data, n_bytes);
    uint8_t* droot = st.out(root32_out, 32);
    if (st.rc) return st.rc;
    uint32_t* tree = ctx->ssz.chunks;
    k_ssz_chunk_leaves<<<blocks_for(C * 8, 256), 256, 0, ctx->s_main>>>(dd, n_bytes, tree, C);
    CKL(ctx);
    if ((rc = ssz_reduce(ctx, tree, C)) || (rc = ssz_root(ctx, tree, C, limit_depth, mix_in != 0, length, droot))) return rc;
    return st.finish();
}

}  // extern "C"
