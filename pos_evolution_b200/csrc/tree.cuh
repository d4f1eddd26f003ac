// tree.cuh -- the fork-choice block tree changed in place on the device: blocks appended (on_block, pos-evolution.md:1015-1018), the
// tree pruned to the finalized block (:1033-1036), leaf viability changed (get_filtered_block_tree, :1104), and the latest messages
// re-mapped through a prune's id map.
//
// Per block id the device keeps the parent, the 32-byte root, the slot, the viability byte, the pre-order position, the subtree size and
// the rank of (root, id) among all blocks -- the order b2_tree_load sorts by.  The slot is read by the attestation intake (intake.cuh).  Siblings are in id order in the pre-order, and an appended block
// has the largest id so far, so it becomes the LAST child of its parent: it takes position pos = pre[p] + size[p], every position
// >= pos moves up by one, and the ancestors of p (p included) are exactly the blocks q with pre[q] <= pre[p] < pre[q] + size[q].
// After every change k_tree_emit re-writes the tables of the tree's kernel form (kernels.cuh ghost_tree_args) from the per-id state.
#pragma once
#include "kernels.cuh"

namespace b2 {

constexpr uint32_t TREE_DROPPED = 0xffffffffu;      // the prune map's value for a block outside the kept subtree

// Appends the blocks n0 .. n0 + k - 1 (parents in `parent`) one after the other in ONE CTA: one pass over the blocks per insertion.
// For trees of the shared-memory form (<= 14 463 blocks), where a pass is a few strided loads per thread.
__global__ void __launch_bounds__(1024) k_tree_insert_cta(uint32_t* pre, uint32_t* size, const uint32_t* parent, uint32_t n0, uint32_t k) {
    __shared__ uint32_t s_p, s_pos;
    for (uint32_t j = 0; j < k; j++) {
        const uint32_t x = n0 + j;
        if (threadIdx.x == 0) {
            const uint32_t p = parent[x];
            s_p = pre[p];
            s_pos = pre[p] + size[p];
        }
        __syncthreads();
        const uint32_t P = s_p, pos = s_pos;
        for (uint32_t q = threadIdx.x; q < x; q += blockDim.x) {
            const uint32_t pq = pre[q];
            if (pq >= pos) pre[q] = pq + 1;
            else if (pq <= P && P < pq + size[q]) size[q] += 1;      // an ancestor lies before pos, a shifted block after it
        }
        if (threadIdx.x == 0) {
            pre[x] = pos;
            size[x] = 1;
        }
        __syncthreads();
    }
}

// One insertion of block x under p over a grid (the generic form): sizes go from size_in to size_out, because p's own size changes while
// other CTAs still read it.  pre[p] itself never moves (it lies before pos), so positions are updated in place.
__global__ void k_tree_insert_grid(uint32_t* pre, const uint32_t* size_in, uint32_t* size_out, uint32_t p, uint32_t x) {
    const uint32_t q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q > x) return;
    const uint32_t P = pre[p], pos = P + size_in[p];
    if (q == x) {
        pre[x] = pos;
        size_out[x] = 1;
        return;
    }
    const uint32_t pq = pre[q], sq = size_in[q];
    if (pq >= pos) pre[q] = pq + 1;
    size_out[q] = sq + (pq <= P && P < pq + sq ? 1u : 0u);
}

// (root, id) order of blocks a and b: the 32-byte roots compared as bytes, then the ids
__device__ __forceinline__ bool tree_key_less(const uint8_t* roots, uint32_t a, uint32_t b) {
    const uint4* ra = reinterpret_cast<const uint4*>(roots + 32ull * a);
    const uint4* rb = reinterpret_cast<const uint4*>(roots + 32ull * b);
#pragma unroll
    for (int h = 0; h < 2; h++) {
        const uint4 x = __ldg(ra + h), y = __ldg(rb + h);
        const uint32_t xs[4] = {x.x, x.y, x.z, x.w}, ys[4] = {y.x, y.y, y.z, y.w};
#pragma unroll
        for (int i = 0; i < 4; i++) {
            const uint32_t u = __byte_perm(xs[i], 0, 0x0123), v = __byte_perm(ys[i], 0, 0x0123);      // big-endian: memcmp order
            if (u != v) return u < v;
        }
    }
    return a < b;
}

// ranks after appending n0 .. n1 - 1: an existing block moves up by the number of new blocks that sort before it
__global__ void k_tree_rank_old(const uint8_t* roots, uint32_t* rank, uint32_t n0, uint32_t n1) {
    const uint32_t q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= n0) return;
    uint32_t c = 0;
    for (uint32_t x = n0; x < n1; x++) c += tree_key_less(roots, x, q);
    if (c) rank[q] += c;
}

// ... and a new block's rank is the number of blocks (old and new) that sort before it: one CTA per new block
__global__ void __launch_bounds__(256) k_tree_rank_new(const uint8_t* roots, uint32_t* rank, uint32_t n0, uint32_t n1) {
    __shared__ uint32_t warp_sum[8];
    const uint32_t x = n0 + blockIdx.x;
    uint32_t c = 0;
    for (uint32_t b = threadIdx.x; b < n1; b += blockDim.x) c += tree_key_less(roots, b, x);
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) c += __shfl_down_sync(B2_FULL_MASK, c, d);
    if ((threadIdx.x & 31) == 0) warp_sum[threadIdx.x >> 5] = c;
    __syncthreads();
    if (threadIdx.x == 0) {
        uint32_t t = 0;
        for (int w = 0; w < 8; w++) t += warp_sum[w];
        rank[x] = t;
    }
}

// the viability bytes of k blocks, in order (a repeated index keeps its last value).  One thread: a call carries the few leaves whose
// test changed since the last one (at most the tree's leaves when a checkpoint moves), and in order is what makes a repeated index
// deterministic.
__global__ void k_tree_set_viable(uint8_t* viable, const uint32_t* idx, const uint8_t* val, uint32_t k) {
    for (uint32_t j = 0; j < k; j++) viable[idx[j]] = val[j];
}

// The tables of the tree's form from the per-id state, in one CTA: inv, and the keep bit of every block from a prefix count of viable
// leaves (size 1) over pre-order positions -- a block is kept iff its interval [pre, pre + size) holds one.  packed != null: the
// shared-memory form (size | rank << 15 | keep << 31), else the generic form's size_keep and rank_p.  cnt: u32[n + 1] scratch.
__global__ void __launch_bounds__(1024) k_tree_emit(const uint32_t* pre, const uint32_t* size, const uint32_t* rank, const uint8_t* viable, uint32_t n,
                                                    uint32_t* cnt, uint32_t* inv, uint32_t* packed, uint32_t* size_keep, uint32_t* rank_p) {
    __shared__ uint32_t warp_tot[32];
    for (uint32_t b = threadIdx.x; b < n; b += blockDim.x) {
        const uint32_t p = pre[b];
        inv[p] = b;
        cnt[p] = size[b] == 1 && viable[b] ? 1u : 0u;
    }
    __syncthreads();
    block_exclusive_scan(cnt, n, warp_tot);
    for (uint32_t b = threadIdx.x; b < n; b += blockDim.x) {
        const uint32_t p = pre[b], s = size[b], keep = cnt[p + s] > cnt[p] ? 0x80000000u : 0u;
        if (packed) {
            packed[p] = s | (rank[b] << 15) | keep;
        } else {
            size_keep[p] = s | keep;
            rank_p[p] = rank[b];
        }
    }
}

struct tree_ids {
    uint32_t *pre, *size, *rank, *parent;
    uint8_t *root, *viable;
    uint64_t* slot;
};

// Prune to the subtree of block r, in one CTA: the kept blocks are those in r's interval of pre-order positions; their new ids are a
// prefix count of kept ids (order-preserving, so parents still precede children), their new ranks a prefix count of kept ranks, and
// their positions move down by pre[r].  Writes the compacted per-id state to `to` and map[old] = new id or TREE_DROPPED.
// kid, krank: u32[n + 1] scratch.
__global__ void __launch_bounds__(1024) k_tree_prune(tree_ids from, tree_ids to, uint32_t n, uint32_t r, uint32_t* kid, uint32_t* krank, uint32_t* map) {
    __shared__ uint32_t warp_tot[32];
    const uint32_t R = from.pre[r], S = from.size[r];
    for (uint32_t b = threadIdx.x; b < n; b += blockDim.x) {
        const uint32_t kept = from.pre[b] - R < S ? 1u : 0u;
        kid[b] = kept;
        krank[from.rank[b]] = kept;
    }
    __syncthreads();
    block_exclusive_scan(kid, n, warp_tot);
    block_exclusive_scan(krank, n, warp_tot);
    for (uint32_t b = threadIdx.x; b < n; b += blockDim.x) {
        const uint32_t p = from.pre[b];
        if (p - R >= S) {
            map[b] = TREE_DROPPED;
            continue;
        }
        const uint32_t nb = kid[b];
        map[b] = nb;
        to.pre[nb] = p - R;
        to.size[nb] = from.size[b];
        to.rank[nb] = krank[from.rank[b]];
        to.parent[nb] = b == r ? 0u : kid[from.parent[b]];
        to.viable[nb] = from.viable[b];
        to.slot[nb] = from.slot[b];
        const uint4* src = reinterpret_cast<const uint4*>(from.root + 32ull * b);
        uint4* dst = reinterpret_cast<uint4*>(to.root + 32ull * nb);
        dst[0] = src[0];
        dst[1] = src[1];
    }
}

// Every validator's latest-message block through a prune's map; a block >= the old size (no such block) stays as it is, and a dropped
// block becomes TREE_DROPPED, which latest_message_counts ignores (block >= n_blocks).  The message keys are not touched.
__global__ void k_lmd_remap(uint32_t* lmd_block, uint64_t n_val, const uint32_t* __restrict__ map, uint32_t n_old) {
    const uint64_t v = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= n_val) return;
    const uint32_t b = lmd_block[v];
    if (b < n_old) lmd_block[v] = map[b];
}

}  // namespace b2
