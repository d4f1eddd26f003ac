// aggverify_sim.cpp -- TEST-ONLY host build of the bls.AggregateVerify bodies (pos_evolution_b200/csrc/cores.cuh), compiled with g++
// by tests/test_hostsim_aggregate_verify.py into a temporary directory; the carry-chain primitives are emulated (csrc/platform.cuh),
// everything above them is the code the kernels of csrc/aggverify.cuh run.  Never linked into, or loaded by, the product.
#include <stddef.h>

#include "cores.cuh"

using namespace b2;

// bls.AggregateVerify with explicit keys: the item loop of k_av_miller (item -> set by av_set_of, the same per-item bodies and one
// Miller loop per item) and the per-set product + verdict of k_av_final, on the host
extern "C" void hs_core_aggregate_verify(const uint8_t* pk48, const uint8_t* msg32, const uint32_t* pair_off, const uint8_t* sig96, uint32_t n_sets,
                                         uint8_t* ok) {
    const uint32_t n_pairs = pair_off[n_sets];
    uint32_t* records = new uint32_t[24 * (size_t)n_pairs + 1];
    uint8_t* valid = new uint8_t[n_pairs + 1];
    for (uint32_t j = 0; j < n_pairs; j++) core_registry_load(pk48, records, valid, j);
    fp12* F = new fp12[n_sets];
    uint32_t* bad = new uint32_t[n_sets];
    for (uint32_t s = 0; s < n_sets; s++) {
        F[s] = fp12_one();
        bad[s] = 0;
    }
    for (uint32_t i = 0; i < n_pairs + n_sets; i++) {
        const uint32_t s = av_set_of(pair_off, n_sets, i), j = i - s;
        g1_jac p;
        g2_aff q;
        bool q_inf;
        if (j < pair_off[s + 1]) {
            g2_aff h;
            uint8_t hflag;
            core_hash_msg(msg32, j, h, hflag);
            core_av_pair(records, valid, j, n_pairs, h, hflag, p, q, q_inf, bad[s]);
        } else {
            g2_aff sg;
            uint8_t sflag;
            core_sig_prepare(sig96, s, sg, sflag);
            core_av_sig(sg, sflag, p, q, q_inf, bad[s]);
        }
        F[s] = fp12_mul(F[s], miller_loop(p, q, q_inf));
    }
    for (uint32_t s = 0; s < n_sets; s++) ok[s] = core_av_verdict(F[s], bad[s], pair_off[s + 1] > pair_off[s]);
    delete[] records;
    delete[] valid;
    delete[] F;
    delete[] bad;
}
