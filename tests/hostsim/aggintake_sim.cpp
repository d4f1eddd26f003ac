// aggintake_sim.cpp -- TEST-ONLY: the SSZ roots and aggregator selection of csrc/aggintake.cuh compiled for the host CPU
// (tests/test_hostsim_aggregate_intake.py)
#include <stddef.h>
#include <stdint.h>

#include "aggintake.cuh"

extern "C" {

// n items: aggregator u64, bit row (stride bytes, nbits bits), data 128, aggregate signature 96, selection proof 96, slot u64 ->
// hash_tree_root(AggregateAndProof), compute_signing_root(Slot(slot), dom) and compute_signing_root(AggregateAndProof, dom), 32 bytes each
void hs_aggregate_and_proof_roots(const uint64_t* aggregator, const uint8_t* rows, uint32_t stride, const uint32_t* nbits, const uint8_t* data128,
                                  const uint8_t* sig96, const uint8_t* proof96, const uint8_t* dom_sel, const uint8_t* dom_aap, uint64_t n,
                                  uint8_t* aap_root32, uint8_t* slot_root32, uint8_t* aap_signing32) {
    for (uint64_t i = 0; i < n; i++) {
        uint8_t le[8], dr[32];
        for (int k = 0; k < 8; k++) le[k] = (uint8_t)(aggregator[i] >> (8 * k));
        b2::attestation_data_root(data128 + 128 * i, dr);
        uint32_t ar[8], pr[8];
        b2::api_attestation_root(rows + stride * i, stride, nbits[i], dr, sig96 + 96 * i, ar);
        b2::api_aggregate_and_proof_root(le, ar, proof96 + 96 * i, pr);
        b2::ssz_store_root(pr, aap_root32 + 32 * i);
        b2::api_signing_root(pr, dom_aap, aap_signing32 + 32 * i);
        b2::api_slot_signing_root(data128 + 128 * i, dom_sel, slot_root32 + 32 * i);
    }
}

// is_aggregator of n selection proofs against committee sizes
void hs_is_aggregator(const uint8_t* proof96, const uint32_t* committee_size, uint32_t target, uint64_t n, uint8_t* out) {
    for (uint64_t i = 0; i < n; i++) out[i] = b2::api_is_aggregator(proof96 + 96 * i, committee_size[i], target) ? 1 : 0;
}

}  // extern "C"
