// ssz.cuh -- hash_tree_root merkleization on the device: SHA-256 of 64-byte tree nodes, the Validator leaf (pos-evolution.md:36-45),
// subtree reductions and the incremental path update of a device-resident tree (SURVEY.md section 8(f)-3, "batch SHA-256 merkleization").
//
// Tree nodes are kept as 8 u32 digest words (SHA-256's big-endian word order), so a parent's 16 input words are its children's 8 + 8
// output words with no byte swap.  Bytes are swapped only where a data chunk enters the tree (ssz_be32) and where a root leaves it
// (ssz_store_root).  A node cache over C leaves (C a power of two) is a heap: node 1 the root, node i's children 2i and 2i + 1, leaves at
// C .. 2C - 1; index 0 is unused.
#pragma once
#include "h2c.cuh"

namespace b2 {

constexpr int SSZ_MAX_DEPTH = 64;              // zero-hash levels a root can be padded through
constexpr uint32_t SSZ_VALIDATOR_BYTES = 121;  // SSZ serialisation of Validator
constexpr int SSZ_SUBTREE_LEVELS = 9;          // k_ssz_subtree: 512 nodes -> 1 per CTA
constexpr int SSZ_LEAF_THREADS = 128;

// zero[l] = root of 2^l zero chunks, in word order
struct ssz_zero_hashes {
    uint32_t z[SSZ_MAX_DEPTH][8];
};

// K[i] + W[i] of SHA-256's second block for a 64-byte message: 0x80000000, fourteen zero words, the bit length 512, expanded.  The
// block never changes, so its compression does no schedule work.
HD uint32_t sha_pad64_kw(int i) {
    constexpr uint32_t KW[64] = {
        0xc28a2f98, 0x71374491, 0xb5c0fbcf, 0xe9b5dba5, 0x3956c25b, 0x59f111f1, 0x923f82a4, 0xab1c5ed5,
        0xd807aa98, 0x12835b01, 0x243185be, 0x550c7dc3, 0x72be5d74, 0x80deb1fe, 0x9bdc06a7, 0xc19bf374,
        0x649b69c1, 0xf0fe4786, 0x0fe1edc6, 0x240cf254, 0x4fe9346f, 0x6cc984be, 0x61b9411e, 0x16f988fa,
        0xf2c65152, 0xa88e5a6d, 0xb019fc65, 0xb9d99ec7, 0x9a1231c3, 0xe70eeaa0, 0xfdb1232b, 0xc7353eb0,
        0x3069bad5, 0xcb976d5f, 0x5a0f118f, 0xdc1eeefd, 0x0a35b689, 0xde0b7a04, 0x58f4ca9d, 0xe15d5b16,
        0x007f3e86, 0x37088980, 0xa507ea32, 0x6fab9537, 0x17406110, 0x0d8cd6f1, 0xcdaa3b6d, 0xc0bbbe37,
        0x83613bda, 0xdb48a363, 0x0b02e931, 0x6fd15ca7, 0x521afaca, 0x31338431, 0x6ed41a95, 0x6d437890,
        0xc39c91f2, 0x9eccabbd, 0xb5c9a0e6, 0x532fb63c, 0xd2c741c6, 0x07237ea3, 0xa4954b68, 0x4c191d76};
    return KW[i];
}

// one SHA-256 round on s[0..7] = a..h with k + w = kw
HD void sha_round(uint32_t* s, uint32_t kw) {
    const uint32_t e = s[4], a = s[0];
    const uint32_t t1 = s[7] + (sha_rotr(e, 6) ^ sha_rotr(e, 11) ^ sha_rotr(e, 25)) + ((e & s[5]) ^ (~e & s[6])) + kw;
    const uint32_t t2 = (sha_rotr(a, 2) ^ sha_rotr(a, 13) ^ sha_rotr(a, 22)) + ((a & s[1]) ^ (a & s[2]) ^ (s[1] & s[2]));
    s[7] = s[6]; s[6] = s[5]; s[5] = s[4]; s[4] = s[3] + t1; s[3] = s[2]; s[2] = s[1]; s[1] = s[0]; s[0] = t1 + t2;
}

// SHA-256 of one 64-byte node given as 16 big-endian words -> 8 digest words
HD void sha256_node(const uint32_t in[16], uint32_t out[8]) {
    uint32_t w[16], s[8];
    const uint32_t iv[8] = {0x6a09e667, 0xbb67ae85, 0x3c6ef372, 0xa54ff53a, 0x510e527f, 0x9b05688c, 0x1f83d9ab, 0x5be0cd19};
#pragma unroll
    for (int i = 0; i < 16; i++) w[i] = in[i];
#pragma unroll
    for (int i = 0; i < 8; i++) s[i] = iv[i];
#pragma unroll
    for (int i = 0; i < 64; i++) {
        if (i >= 16) {      // rolling 16-word schedule: w[i & 15] becomes W[i]
            const uint32_t w15 = w[(i - 15) & 15], w2 = w[(i - 2) & 15];
            w[i & 15] += (sha_rotr(w15, 7) ^ sha_rotr(w15, 18) ^ (w15 >> 3)) + w[(i - 7) & 15] + (sha_rotr(w2, 17) ^ sha_rotr(w2, 19) ^ (w2 >> 10));
        }
        sha_round(s, sha_k(i) + w[i & 15]);
    }
    uint32_t h[8];
#pragma unroll
    for (int i = 0; i < 8; i++) h[i] = s[i] += iv[i];
#pragma unroll
    for (int i = 0; i < 64; i++) sha_round(s, sha_pad64_kw(i));
#pragma unroll
    for (int i = 0; i < 8; i++) out[i] = h[i] + s[i];
}

HD void sha256_node_pair(const uint32_t* l, const uint32_t* r, uint32_t* out) {
    uint32_t in[16];
#pragma unroll
    for (int i = 0; i < 8; i++) in[i] = l[i], in[8 + i] = r[i];
    sha256_node(in, out);
}

HD uint32_t ssz_be32(const uint8_t* p) { return ((uint32_t)p[0] << 24) | ((uint32_t)p[1] << 16) | ((uint32_t)p[2] << 8) | p[3]; }

// the chunk of a little-endian u64 at p (8 bytes, then 24 zero bytes), in word order
HD void ssz_u64_chunk(const uint8_t* p, uint32_t* c) {
    c[0] = ssz_be32(p);
    c[1] = ssz_be32(p + 4);
#pragma unroll
    for (int i = 2; i < 8; i++) c[i] = 0;
}

HD void ssz_store_root(const uint32_t* h, uint8_t* out32) {
#pragma unroll
    for (int i = 0; i < 8; i++) {
        out32[4 * i] = (uint8_t)(h[i] >> 24);
        out32[4 * i + 1] = (uint8_t)(h[i] >> 16);
        out32[4 * i + 2] = (uint8_t)(h[i] >> 8);
        out32[4 * i + 3] = (uint8_t)h[i];
    }
}

// hash_tree_root(Validator) of its 121-byte serialisation: pubkey 48, withdrawal_credentials 32, effective_balance u64, slashed 1,
// activation_eligibility_epoch, activation_epoch, exit_epoch, withdrawable_epoch u64 (little-endian).  Chunks: the pubkey's root
// H(pk[0:32] || pk[32:48] || 0^16), the credentials, then one padded chunk per basic field; the 8 chunks reduce in 7 node hashes.
HD void ssz_validator_root(const uint8_t* r, uint32_t out[8]) {
    uint32_t in[16], a[8], b[8], l1[4][8];
#pragma unroll
    for (int i = 0; i < 12; i++) in[i] = ssz_be32(r + 4 * i);
#pragma unroll
    for (int i = 12; i < 16; i++) in[i] = 0;
    sha256_node(in, a);                                   // pubkey root
#pragma unroll
    for (int i = 0; i < 8; i++) b[i] = ssz_be32(r + 48 + 4 * i);
    sha256_node_pair(a, b, l1[0]);
    ssz_u64_chunk(r + 80, a);                             // effective_balance
#pragma unroll
    for (int i = 0; i < 8; i++) b[i] = 0;
    b[0] = (uint32_t)r[88] << 24;                         // slashed
    sha256_node_pair(a, b, l1[1]);
#pragma unroll
    for (int j = 0; j < 2; j++) {                         // the four epochs
        ssz_u64_chunk(r + 89 + 16 * j, a);
        ssz_u64_chunk(r + 97 + 16 * j, b);
        sha256_node_pair(a, b, l1[2 + j]);
    }
    sha256_node_pair(l1[0], l1[1], a);
    sha256_node_pair(l1[2], l1[3], b);
    sha256_node_pair(a, b, out);
}

#if defined(__CUDACC__)
// The leaves of a validators tree: record j of rec (k records of 121 bytes) is leaf idx[j] (j when idx is null) of the cache over C
// leaves.  The CTA's records are staged through shared memory with coalesced word loads; rec must be 4-byte aligned.
__global__ void __launch_bounds__(SSZ_LEAF_THREADS) k_ssz_validator_leaves(const uint8_t* __restrict__ rec, const uint32_t* __restrict__ idx,
                                                                           uint64_t k, uint32_t* __restrict__ cache, uint64_t C) {
    __shared__ uint32_t s[SSZ_LEAF_THREADS * SSZ_VALIDATOR_BYTES / 4];
    const uint64_t first = (uint64_t)blockIdx.x * SSZ_LEAF_THREADS;
    const uint32_t cnt = (uint32_t)(k - first < SSZ_LEAF_THREADS ? k - first : SSZ_LEAF_THREADS), bytes = cnt * SSZ_VALIDATOR_BYTES;
    const uint8_t* src = rec + first * SSZ_VALIDATOR_BYTES;
    for (uint32_t w = threadIdx.x; w < bytes / 4; w += blockDim.x) s[w] = reinterpret_cast<const uint32_t*>(src)[w];
    uint8_t* sb = reinterpret_cast<uint8_t*>(s);
    if (threadIdx.x < bytes % 4) sb[bytes / 4 * 4 + threadIdx.x] = src[bytes / 4 * 4 + threadIdx.x];
    __syncthreads();
    if (threadIdx.x >= cnt) return;
    uint32_t h[8];
    ssz_validator_root(sb + threadIdx.x * SSZ_VALIDATOR_BYTES, h);
    const uint64_t j = first + threadIdx.x;
    uint4* dst = reinterpret_cast<uint4*>(cache + (C + (idx ? idx[j] : j)) * 8);
    dst[0] = make_uint4(h[0], h[1], h[2], h[3]);
    dst[1] = make_uint4(h[4], h[5], h[6], h[7]);
}

// The C leaves of a chunk tree from n_bytes of data: 32-byte chunks, the last one zero-padded, then zero chunks.  One thread per word.
__global__ void k_ssz_chunk_leaves(const uint8_t* __restrict__ data, uint64_t n_bytes, uint32_t* __restrict__ cache, uint64_t C) {
    const uint64_t w = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (w >= C * 8) return;
    uint32_t v = 0;
#pragma unroll
    for (int i = 0; i < 4; i++) {
        const uint64_t b = 4 * w + i;
        v = v << 8 | (b < n_bytes ? data[b] : 0u);
    }
    cache[C * 8 + w] = v;
}

// One CTA reduces the 2^levels nodes m + blockIdx.x * 2^levels ... of heap level m (m nodes) through `levels` levels, writing every
// level it computes into the cache.  The first level reads its children from the cache, the later ones from shared memory.
__global__ void __launch_bounds__(256) k_ssz_subtree(uint32_t* __restrict__ cache, uint64_t m, uint32_t levels) {
    __shared__ uint4 node[256][2];
    const uint32_t t = threadIdx.x;
#pragma unroll 1
    for (uint32_t j = 0; j < levels; j++) {
        const uint32_t half = 1u << (levels - 1 - j);      // parents this level computes
        uint32_t in[16], h[8];
        if (t < half) {
            const uint4* c = j == 0 ? reinterpret_cast<const uint4*>(cache + ((m + ((uint64_t)blockIdx.x << levels)) + 2 * t) * 8) : node[2 * t];
#pragma unroll
            for (int q = 0; q < 4; q++) {
                const uint4 v = c[q];
                in[4 * q] = v.x, in[4 * q + 1] = v.y, in[4 * q + 2] = v.z, in[4 * q + 3] = v.w;
            }
            sha256_node(in, h);
        }
        __syncthreads();      // every read of this level's children before any parent overwrites them
        if (t < half) {
            const uint4 lo = make_uint4(h[0], h[1], h[2], h[3]), hi = make_uint4(h[4], h[5], h[6], h[7]);
            node[t][0] = lo, node[t][1] = hi;
            uint4* dst = reinterpret_cast<uint4*>(cache + ((m >> (j + 1)) + ((uint64_t)blockIdx.x << (levels - 1 - j)) + t) * 8);
            dst[0] = lo, dst[1] = hi;
        }
        __syncthreads();
    }
}

// One level of an incremental update: leaves C + idx[t] (idx sorted, unique) were re-hashed; their ancestors `shift` levels up are
// re-hashed from their children.  Sorted indices put equal parents next to each other, so the first thread of each run hashes it.
__global__ void k_ssz_update_level(uint32_t* __restrict__ cache, const uint32_t* __restrict__ idx, uint64_t k, uint64_t C, uint32_t shift) {
    const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= k) return;
    const uint64_t p = (C + idx[t]) >> shift;
    if (t > 0 && ((C + idx[t - 1]) >> shift) == p) return;
    uint32_t h[8];
    sha256_node(cache + 2 * p * 8, h);
    uint4* dst = reinterpret_cast<uint4*>(cache + p * 8);
    dst[0] = make_uint4(h[0], h[1], h[2], h[3]);
    dst[1] = make_uint4(h[4], h[5], h[6], h[7]);
}

// The root of a tree whose top (node 1 of the cache, a subtree of depth `level`) is padded with zero subtrees up to depth `depth`,
// then, when mix_in is set, mix_in_length(root, length).  One thread: the chain is serial.
__global__ void k_ssz_root(const uint32_t* __restrict__ top, uint32_t level, uint32_t depth, ssz_zero_hashes Z, int mix_in, uint64_t length,
                           uint8_t* __restrict__ out32) {
    if (threadIdx.x) return;
    uint32_t r[8], c[8];
#pragma unroll
    for (int i = 0; i < 8; i++) r[i] = top[i];
#pragma unroll 1
    for (uint32_t l = level; l < depth; l++) {
        sha256_node_pair(r, Z.z[l], c);
#pragma unroll
        for (int i = 0; i < 8; i++) r[i] = c[i];
    }
    if (mix_in) {
        uint8_t le[8];
#pragma unroll
        for (int i = 0; i < 8; i++) le[i] = (uint8_t)(length >> (8 * i));
        ssz_u64_chunk(le, c);
        sha256_node_pair(r, c, r);
    }
    ssz_store_root(r, out32);
}
#endif

}  // namespace b2
