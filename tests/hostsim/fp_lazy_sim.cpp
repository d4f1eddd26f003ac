// fp_lazy_sim.cpp -- TEST-ONLY host build of the lazily reduced Fp forms (pos_evolution_b200/csrc/fp.cuh) and of the fixed-exponent
// chain that runs on them, compiled with g++ by tests/test_hostsim_fp_lazy.py into a temporary directory.  The carry-chain primitives
// are emulated (csrc/platform.cuh); everything above them is the code the kernels run.  Never linked into, or loaded by, the product.
#include <string.h>

#include "fp.cuh"

using namespace b2;

static fp ld(const uint32_t* p) {
    fp v;
    memcpy(&v, p, sizeof(fp));
    return v;
}
static void st(uint32_t* p, const fp& v) { memcpy(p, &v, sizeof(fp)); }

extern "C" {
void hs_fp_mul_lazy(const uint32_t* a, const uint32_t* b, uint32_t* r) { st(r, fp_mul_lazy(ld(a), ld(b))); }
void hs_fp_sqr_lazy(const uint32_t* a, uint32_t* r) { st(r, fp_sqr_lazy(ld(a))); }
void hs_fp_mul(const uint32_t* a, const uint32_t* b, uint32_t* r) { st(r, fp_mul(ld(a), ld(b))); }
void hs_fp_sqr(const uint32_t* a, uint32_t* r) { st(r, fp_sqr(ld(a))); }
// which = 0: a^((p-3)/4), 1: a^(p-2)
void hs_fp_pow_prog(const uint32_t* a, int which, uint32_t* r) { st(r, fp_pow_prog(ld(a), which ? C_PROG_PM2 : C_PROG_PM3D4)); }
}
