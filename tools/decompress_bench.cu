// decompress_bench.cu -- timing harness for the G2 decompression kernel body (two Fp exponentiations per signature, window tables in
// local memory), compiled against whichever csrc/ tree -I points to (A/B of two trees, or of -DB2_SIG_VECTOR_LOADS).
// Inputs: 2^20 valid compressed G2 points (x = 1 + k*u scanned until on-curve), so both exponentiations run for every thread.
// Build: nvcc -O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a -I pos_evolution_b200/csrc -o tools/decompress_bench.bin tools/decompress_bench.cu
#include <cstdio>
#include <cstdlib>
#include <vector>
#include <cuda_runtime.h>
#include "cores.cuh"
using namespace b2;

__global__ void __launch_bounds__(128, 4) k_dec(const uint8_t* __restrict__ sig96, uint64_t n, uint32_t* aff_out, uint8_t* st_out) {
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

int main() {
    const uint64_t want = 1u << 20, cand = 5u << 19;
    std::vector<uint8_t> h(cand * 96, 0);
    uint64_t x = 0x243f6a8885a308d3ull;
    for (uint64_t i = 0; i < cand; i++) {
        uint8_t* p = h.data() + 96 * i;
        for (int k = 8; k < 96; k++) {
            x ^= x << 13; x ^= x >> 7; x ^= x << 17;
            p[k] = (uint8_t)(x >> 17);
        }
        p[0] = 0x80 | (uint8_t)(i & 0x20 ? 0x20 : 0);          // compressed, random sign, top bits of x.c1 zero (x.c1 < p)
        p[48] = 0;                                              // x.c0 < p
    }
    uint8_t *d_sig, *d_st;
    uint32_t* d_aff;
    cudaMalloc(&d_sig, cand * 96);
    cudaMalloc(&d_st, cand);
    cudaMalloc(&d_aff, cand * 192);
    cudaMemcpy(d_sig, h.data(), cand * 96, cudaMemcpyHostToDevice);
    k_dec<<<(unsigned)((cand + 127) / 128), 128>>>(d_sig, cand, d_aff, d_st);
    std::vector<uint8_t> st(cand);
    cudaMemcpy(st.data(), d_st, cand, cudaMemcpyDeviceToHost);
    std::vector<uint8_t> good(want * 96);
    uint64_t n = 0;
    for (uint64_t i = 0; i < cand && n < want; i++)
        if (st[i] == 0) memcpy(good.data() + 96 * n++, h.data() + 96 * i, 96);
    if (n < want) {
        printf("{\"error\": \"only %llu valid points\"}\n", (unsigned long long)n);
        return 1;
    }
    cudaMemcpy(d_sig, good.data(), want * 96, cudaMemcpyHostToDevice);
    cudaEvent_t e0, e1;
    cudaEventCreate(&e0);
    cudaEventCreate(&e1);
    float best = 1e9f, sum = 0;
    const int reps = 6;
    for (int r = 0; r < reps + 1; r++) {
        cudaEventRecord(e0);
        k_dec<<<(unsigned)(want / 128), 128>>>(d_sig, want, d_aff, d_st);
        cudaEventRecord(e1);
        cudaDeviceSynchronize();
        float ms;
        cudaEventElapsedTime(&ms, e0, e1);
        if (r) {
            best = ms < best ? ms : best;
            sum += ms;
        }
    }
    cudaMemcpy(st.data(), d_st, want, cudaMemcpyDeviceToHost);
    uint64_t ok = 0;
    for (uint64_t i = 0; i < want; i++) ok += st[i] == 0;
    std::vector<uint32_t> aff(48 * 16);
    cudaMemcpy(aff.data(), d_aff, aff.size() * 4, cudaMemcpyDeviceToHost);
    uint32_t chk = 0;
    for (uint32_t w : aff) chk = chk * 31 + w;
    printf("{\"n\": %llu, \"valid\": %llu, \"ms_mean\": %.3f, \"ms_best\": %.3f, \"checksum\": %u, \"cuda\": \"%s\"}\n", (unsigned long long)want,
           (unsigned long long)ok, sum / reps, best, chk, cudaGetErrorString(cudaGetLastError()));
    return 0;
}
