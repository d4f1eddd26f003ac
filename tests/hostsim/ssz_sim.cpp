// ssz_sim.cpp -- TEST-ONLY: the node hash and the Validator leaf of csrc/ssz.cuh compiled for the host CPU (tests/test_hostsim_ssz.py)
#include <stddef.h>
#include <stdint.h>

#include "ssz.cuh"

extern "C" {

// n nodes of 16 big-endian words -> n digests of 8 words
void hs_sha256_node(const uint32_t* in16, uint64_t n, uint32_t* out8) {
    for (uint64_t i = 0; i < n; i++) b2::sha256_node(in16 + 16 * i, out8 + 8 * i);
}

// n records of 121 bytes -> n hash_tree_root(Validator), 32 bytes each
void hs_validator_root(const uint8_t* rec121, uint64_t n, uint8_t* out32) {
    for (uint64_t i = 0; i < n; i++) {
        uint32_t h[8];
        b2::ssz_validator_root(rec121 + i * b2::SSZ_VALIDATOR_BYTES, h);
        b2::ssz_store_root(h, out32 + 32 * i);
    }
}

}  // extern "C"
