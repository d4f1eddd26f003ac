// synccontrib_sim.cpp -- TEST-ONLY: the SSZ roots and aggregator selection of csrc/synccontrib.cuh compiled for the host CPU
// (tests/test_hostsim_sync_contributions.py)
#include <stddef.h>
#include <stdint.h>

#include "synccontrib.cuh"

extern "C" {

// n items of len_i = 344 + sb bytes each, back to back (every field fixed) -> the Bitvector, SyncCommitteeContribution and
// ContributionAndProof roots, and the three signing roots (selection, contribution_and_proof, sync committee domains), 32 bytes each
void hs_sync_contribution_roots(const uint8_t* wire, uint32_t sb, uint64_t n, const uint8_t* dom_sync, const uint8_t* dom_sel, const uint8_t* dom_cap,
                                uint8_t* bits_root32, uint8_t* contribution_root32, uint8_t* cap_root32, uint8_t* sel32, uint8_t* cap32, uint8_t* sync32) {
    for (uint64_t i = 0; i < n; i++) {
        const uint8_t* m = wire + (344 + sb) * i;
        uint32_t r[8];
        b2::scc_bitvector_root(m + b2::SCC_BITS, sb, r);
        b2::ssz_store_root(r, bits_root32 + 32 * i);
        b2::scc_contribution_root(m + b2::SCC_SLOT, sb, r);
        b2::ssz_store_root(r, contribution_root32 + 32 * i);
        b2::scc_contribution_and_proof_root(m, sb, r);
        b2::ssz_store_root(r, cap_root32 + 32 * i);
        b2::scc_signing_roots(m, sb, dom_sel, dom_cap, dom_sync, sel32 + 32 * i, cap32 + 32 * i, sync32 + 32 * i);
    }
}

// is_sync_committee_aggregator of n selection proofs against subcommittee sizes
void hs_sync_is_aggregator(const uint8_t* proof96, const uint32_t* sub, uint32_t target, uint64_t n, uint8_t* out) {
    for (uint64_t i = 0; i < n; i++) out[i] = b2::scc_is_aggregator(proof96 + 96 * i, sub[i], target) ? 1 : 0;
}

}  // extern "C"
