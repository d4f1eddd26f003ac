// platform.cuh -- compile-target glue for the BLS12-381 device library.
//
// Every arithmetic routine in csrc/*.cuh is written once as `HD` (host+device) code on top of
// the twelve carry-chain primitives below.  Under nvcc for sm_90a they are single PTX
// instructions using the hardware carry flag (add.cc / madc.hi.cc ...; ptxas fuses the
// mad.lo.cc+madc.hi.cc pairs into IMAD.WIDE.U32 with a predicate carry).  Compiled by a plain
// host compiler (tests/hostsim only -- never part of the product library) the same
// primitives are emulated with an explicit carry variable, so the whole algorithm layer
// (field towers, curve ops, hash-to-curve, pairing) is unit-tested against the oracle on a
// machine without a GPU.  The product (libb200pos.so) only ever runs the PTX path.
#pragma once
#include <stdint.h>

#if defined(__CUDACC__)
#define HD __host__ __device__ __forceinline__
#define HDN __host__ __device__ __noinline__
#define DEV __device__ __forceinline__
#else
#define HD inline
#define HDN inline
#define DEV inline
#endif

namespace b2 {

#if defined(__CUDA_ARCH__)
// ---------------------------------------------------------------- device: PTX with hardware carry
DEV uint32_t add_cc(uint32_t a, uint32_t b) { uint32_t r; asm volatile("add.cc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
DEV uint32_t addc_cc(uint32_t a, uint32_t b) { uint32_t r; asm volatile("addc.cc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
DEV uint32_t addc(uint32_t a, uint32_t b) { uint32_t r; asm volatile("addc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
DEV uint32_t sub_cc(uint32_t a, uint32_t b) { uint32_t r; asm volatile("sub.cc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
DEV uint32_t subc_cc(uint32_t a, uint32_t b) { uint32_t r; asm volatile("subc.cc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
DEV uint32_t subc(uint32_t a, uint32_t b) { uint32_t r; asm volatile("subc.u32 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b)); return r; }
DEV uint32_t mul_lo(uint32_t a, uint32_t b) { return a * b; }
DEV uint32_t mul_hi(uint32_t a, uint32_t b) { return __umulhi(a, b); }
DEV uint32_t mad_lo_cc(uint32_t a, uint32_t b, uint32_t c) { uint32_t r; asm volatile("mad.lo.cc.u32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(c)); return r; }
DEV uint32_t madc_lo_cc(uint32_t a, uint32_t b, uint32_t c) { uint32_t r; asm volatile("madc.lo.cc.u32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(c)); return r; }
DEV uint32_t mad_hi_cc(uint32_t a, uint32_t b, uint32_t c) { uint32_t r; asm volatile("mad.hi.cc.u32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(c)); return r; }
DEV uint32_t madc_hi_cc(uint32_t a, uint32_t b, uint32_t c) { uint32_t r; asm volatile("madc.hi.cc.u32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(c)); return r; }
DEV uint32_t madc_hi(uint32_t a, uint32_t b, uint32_t c) { uint32_t r; asm volatile("madc.hi.u32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(c)); return r; }
// 64-bit-wide multiply-accumulate steps.  The lo/hi halves MUST sit in one asm statement: ptxas only
// fuses adjacent mad.lo.cc + madc.hi.cc into a single IMAD.WIDE.U32(.X) (checked with cuobjdump).
// The plain product is one mul.wide.u32 into a 64-bit register, which is one IMAD.WIDE.U32 by definition; a mul.lo / mul.hi
// pair is one only when ptxas pairs the two (CUDA 12.9 does; otherwise it is an IMAD plus an IMAD.HI.U32, 6 pipe cycles, not 4).
DEV void mul_wide(uint32_t& lo, uint32_t& hi, uint32_t a, uint32_t b) {
    asm("{ .reg .b64 t; mul.wide.u32 t, %2, %3; mov.b64 {%0, %1}, t; }" : "=r"(lo), "=r"(hi) : "r"(a), "r"(b));
}
DEV void mad_wide_cc(uint32_t& lo, uint32_t& hi, uint32_t a, uint32_t b) {          // (hi:lo) += a*b ; CF out
    asm volatile("mad.lo.cc.u32 %0, %2, %3, %0; madc.hi.cc.u32 %1, %2, %3, %1;" : "+r"(lo), "+r"(hi) : "r"(a), "r"(b));
}
DEV void madc_wide_cc(uint32_t& lo, uint32_t& hi, uint32_t a, uint32_t b) {         // (hi:lo) += a*b + CF ; CF out
    asm volatile("madc.lo.cc.u32 %0, %2, %3, %0; madc.hi.cc.u32 %1, %2, %3, %1;" : "+r"(lo), "+r"(hi) : "r"(a), "r"(b));
}
DEV void madc_wide_cc_from(uint32_t& dlo, uint32_t& dhi, uint32_t a, uint32_t b, uint32_t clo, uint32_t chi) {
    asm volatile("madc.lo.cc.u32 %0, %2, %3, %4; madc.hi.cc.u32 %1, %2, %3, %5;" : "=r"(dlo), "=r"(dhi) : "r"(a), "r"(b), "r"(clo), "r"(chi));
}
#else
// ---------------------------------------------------------------- host (tests/hostsim): emulated carry flag
static thread_local uint32_t g_cf = 0;
inline uint32_t emu_add(uint32_t a, uint32_t b, uint32_t cin, bool set) {
    uint64_t s = (uint64_t)a + b + cin;
    if (set) g_cf = (uint32_t)(s >> 32);
    return (uint32_t)s;
}
inline uint32_t emu_sub(uint32_t a, uint32_t b, uint32_t bin, bool set) {
    uint64_t s = (uint64_t)a - b - bin;
    if (set) g_cf = (uint32_t)((s >> 32) & 1);      // PTX: CF holds the borrow for sub.cc / subc
    return (uint32_t)s;
}
inline uint32_t add_cc(uint32_t a, uint32_t b) { return emu_add(a, b, 0, true); }
inline uint32_t addc_cc(uint32_t a, uint32_t b) { return emu_add(a, b, g_cf, true); }
inline uint32_t addc(uint32_t a, uint32_t b) { return emu_add(a, b, g_cf, false); }
inline uint32_t sub_cc(uint32_t a, uint32_t b) { return emu_sub(a, b, 0, true); }
inline uint32_t subc_cc(uint32_t a, uint32_t b) { return emu_sub(a, b, g_cf, true); }
inline uint32_t subc(uint32_t a, uint32_t b) { return emu_sub(a, b, g_cf, false); }
inline uint32_t mul_lo(uint32_t a, uint32_t b) { return a * b; }
inline uint32_t mul_hi(uint32_t a, uint32_t b) { return (uint32_t)(((uint64_t)a * b) >> 32); }
inline uint32_t mad_lo_cc(uint32_t a, uint32_t b, uint32_t c) { return emu_add(a * b, c, 0, true); }
inline uint32_t madc_lo_cc(uint32_t a, uint32_t b, uint32_t c) { return emu_add(a * b, c, g_cf, true); }
inline uint32_t mad_hi_cc(uint32_t a, uint32_t b, uint32_t c) { return emu_add(mul_hi(a, b), c, 0, true); }
inline uint32_t madc_hi_cc(uint32_t a, uint32_t b, uint32_t c) { return emu_add(mul_hi(a, b), c, g_cf, true); }
inline uint32_t madc_hi(uint32_t a, uint32_t b, uint32_t c) { return emu_add(mul_hi(a, b), c, g_cf, false); }
inline void mul_wide(uint32_t& lo, uint32_t& hi, uint32_t a, uint32_t b) { uint64_t p = (uint64_t)a * b; lo = (uint32_t)p; hi = (uint32_t)(p >> 32); }
inline void mad_wide_cc(uint32_t& lo, uint32_t& hi, uint32_t a, uint32_t b) { lo = mad_lo_cc(a, b, lo); hi = madc_hi_cc(a, b, hi); }
inline void madc_wide_cc(uint32_t& lo, uint32_t& hi, uint32_t a, uint32_t b) { lo = madc_lo_cc(a, b, lo); hi = madc_hi_cc(a, b, hi); }
inline void madc_wide_cc_from(uint32_t& dlo, uint32_t& dhi, uint32_t a, uint32_t b, uint32_t clo, uint32_t chi) { dlo = madc_lo_cc(a, b, clo); dhi = madc_hi_cc(a, b, chi); }
#endif

}  // namespace b2
