// blockatt_electra_sim.cpp -- TEST-ONLY: the decode and checks 1-12 of csrc/blockatt_electra.cuh compiled for the host CPU
// (tests/test_hostsim_block_attestations_electra.py)
#include <stddef.h>
#include <stdint.h>

#include "blockatt_electra.cuh"

namespace {
struct one_lane {
    bool operator()(bool x) const { return x; }
};
}  // namespace

extern "C" {

// n attestations wire[woff[i], woff[i+1]) included at bslot[i] in epoch e -> status (checks 1-12), flag mask, Bitlist length, committee_bits
void hs_bae_check(const uint8_t* wire, const uint32_t* woff, uint32_t n, const uint64_t* bslot, uint64_t e, const uint32_t* off, uint64_t n_sig,
                  uint32_t M, uint32_t max_vpc, uint32_t cps_prev, uint32_t cps_cur, uint32_t spe, uint32_t min_delay, uint32_t isqrt_spe,
                  uint32_t row_max, const uint8_t* chain_roots, const uint8_t* justified80, int32_t* status, uint8_t* mask, uint32_t* nbits,
                  uint64_t* cmask) {
    for (uint32_t i = 0; i < n; i++) {
        const b2::bae_in I = {wire + woff[i], (uint64_t)(woff[i + 1] - woff[i]), bslot[i], e, off, n_sig, M, max_vpc, cps_prev, cps_cur, spe,
                              min_delay, isqrt_spe, row_max, chain_roots, justified80};
        b2::bae_out O;
        status[i] = b2::bae_check(I, 0, 1, one_lane{}, O);
        mask[i] = (uint8_t)O.mask;
        nbits[i] = O.nbits;
        cmask[i] = O.cmask;
    }
}

// the OR over lanes 0 .. nl - 1 of bae_any_bit(bl, lo, hi, lane, nl)
int hs_bae_any_bit(const uint8_t* bl, uint32_t lo, uint32_t hi, uint32_t nl) {
    bool any = false;
    for (uint32_t l = 0; l < nl; l++) any |= b2::bae_any_bit(bl, lo, hi, l, nl);
    return any;
}

}  // extern "C"
