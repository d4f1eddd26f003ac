// fp.cuh -- arithmetic in Fp (p = BLS12-381 base field, 381 bits), 12 x 32-bit limbs held in
// registers, Montgomery form with R = 2^384, values fully reduced to [0, p).  The one exception is the
// inside of a fixed-exponent chain (fp_pow_prog_t), whose values stay in [0, 2p) (fp_mul_lazy / fp_sqr_lazy).
//
// This is kernel K1 of SURVEY.md section 2 (no counterpart in the reference: the reference
// reaches field arithmetic only through its bls.* call sites, pos-evolution.md:165/:736/:976).
//
// Montgomery multiplication: word-serial CIOS with two interleaved accumulators.  Products
// a_j*b_i are 64 bits wide and land on limbs (j, j+1); the six even-j products of a row do
// not overlap, nor do the six odd-j products, so each half-row is ONE carry chain of
// mad.lo.cc / madc.hi.cc pairs (ptxas: IMAD.WIDE.U32 with predicate carry).  `ev` collects
// the chain aligned at limb 0, `od` the chain aligned at limb 1; the two chains are
// data-independent, which gives the integer pipe two instructions in flight per thread.
// After the reduction step ev[0] == 0 and the division by 2^32 is a change of roles: the
// old `od` becomes the limb-0 accumulator and the old `ev`, shifted down by two limbs while
// the next row is accumulated into it, becomes the limb-1 accumulator.
#pragma once
#include "consts.cuh"

#ifndef B2_SQR_KARATSUBA
#define B2_SQR_KARATSUBA 0
#endif

namespace b2 {

struct fp {
    uint32_t l[12];
};

HD fp fp_load_const(int off) {
    fp r;
    const uint32_t* t = const_table() + off;
#pragma unroll
    for (int i = 0; i < 12; i++) r.l[i] = t[i];
    return r;
}
HD fp fp_zero() {
    fp r;
#pragma unroll
    for (int i = 0; i < 12; i++) r.l[i] = 0;
    return r;
}
HD fp fp_one() { return fp_load_const(C_ONE); }

HD bool fp_is_zero(const fp& a) {
    uint32_t o = 0;
#pragma unroll
    for (int i = 0; i < 12; i++) o |= a.l[i];
    return o == 0;
}
HD bool fp_eq(const fp& a, const fp& b) {
    uint32_t o = 0;
#pragma unroll
    for (int i = 0; i < 12; i++) o |= a.l[i] ^ b.l[i];
    return o == 0;
}
// branch-free select: c ? a : b
HD fp fp_select(bool c, const fp& a, const fp& b) {
    fp r;
#pragma unroll
    for (int i = 0; i < 12; i++) r.l[i] = c ? a.l[i] : b.l[i];
    return r;
}

// r = (t >= p) ? t - p : t     for t < 2p
HD void fp_final_sub(uint32_t* t) {
    uint32_t d[12];
    d[0] = sub_cc(t[0], P_LIMB(0));
#pragma unroll
    for (int i = 1; i < 12; i++) d[i] = subc_cc(t[i], P_LIMB(i));
    uint32_t borrow = subc(0, 0);               // 0xffffffff when t < p
#pragma unroll
    for (int i = 0; i < 12; i++) t[i] = borrow ? t[i] : d[i];
}

HD fp fp_add(const fp& a, const fp& b) {
    fp r;
    r.l[0] = add_cc(a.l[0], b.l[0]);
#pragma unroll
    for (int i = 1; i < 12; i++) r.l[i] = addc_cc(a.l[i], b.l[i]);
    fp_final_sub(r.l);                          // a + b < 2p < 2^384: no carry out
    return r;
}

HD fp fp_sub(const fp& a, const fp& b) {
    fp r;
    r.l[0] = sub_cc(a.l[0], b.l[0]);
#pragma unroll
    for (int i = 1; i < 12; i++) r.l[i] = subc_cc(a.l[i], b.l[i]);
    uint32_t m = subc(0, 0);                    // all-ones when a < b
    r.l[0] = add_cc(r.l[0], P_LIMB(0) & m);
#pragma unroll
    for (int i = 1; i < 12; i++) r.l[i] = addc_cc(r.l[i], P_LIMB(i) & m);
    return r;
}

HD fp fp_neg(const fp& a) {
    uint32_t nz = 0;
#pragma unroll
    for (int i = 0; i < 12; i++) nz |= a.l[i];
    uint32_t m = nz ? 0xffffffffu : 0u;
    fp r;
    r.l[0] = sub_cc(P_LIMB(0) & m, a.l[0]);
#pragma unroll
    for (int i = 1; i < 12; i++) r.l[i] = subc_cc(P_LIMB(i) & m, a.l[i]);
    return r;
}

HD fp fp_dbl(const fp& a) { return fp_add(a, a); }

// one reduction step: m = E[0]*(-p^-1); (E, O) += m*p; afterwards E[0] == 0
HD void mont_reduce_row(uint32_t* E, uint32_t* O) {
    uint32_t m = E[0] * B2_MONT_INV;
    mad_wide_cc(O[0], O[1], P_LIMB(1), m);
#pragma unroll
    for (int k = 2; k < 12; k += 2) madc_wide_cc(O[k], O[k + 1], P_LIMB(k + 1), m);
    // no carry out of O: the running total is < 2^416 (see fp_mul_lazy)
    mad_wide_cc(E[0], E[1], P_LIMB(0), m);
#pragma unroll
    for (int j = 2; j < 12; j += 2) madc_wide_cc(E[j], E[j + 1], P_LIMB(j), m);
    O[11] = addc(O[11], 0);                     // E's carry out lands on limb 12 = O[11]
}

// accumulate row a*bi.  E: accumulator aligned at limb 0 (the previous row's odd accumulator);
// X: the previous even accumulator (X[0] == 0), rewritten in place as the new odd accumulator.
HD void mont_mul_row(uint32_t* E, uint32_t* X, const uint32_t* a, uint32_t bi) {
    E[0] = add_cc(E[0], X[1]);                  // old limb 1 -> new limb 0; carry goes to new limb 1 = X'[0]
#pragma unroll
    for (int k = 0; k < 12; k += 2)
        madc_wide_cc_from(X[k], X[k + 1], a[k + 1], bi, (k + 2 < 12) ? X[k + 2] : 0u, (k + 3 < 12) ? X[k + 3] : 0u);
    // hi(a*b) <= 2^32-2: the final +carry cannot overflow
    mad_wide_cc(E[0], E[1], a[0], bi);
#pragma unroll
    for (int j = 2; j < 12; j += 2) madc_wide_cc(E[j], E[j + 1], a[j], bi);
    X[11] = addc(X[11], 0);
}

// a*b/R mod p in [0, 2p) for a, b in [0, 2p), without the final subtraction.  With S the running value after a row and its
// division by 2^32, S < a + p by induction (S' < (a + p + (a + p)(2^32 - 1)) / 2^32), so before the division a row holds
// < 3p * 2^32 < 2^416: the 13 limbs of (ev, od) never carry out.  The result is (ab + Mp)/R < 4p^2/R + p < 1.5p (p < R/8).
HD fp fp_mul_lazy(const fp& a, const fp& b) {
    uint32_t ev[12], od[12];
    const uint32_t b0 = b.l[0];
#pragma unroll
    for (int j = 0; j < 12; j += 2) {
        mul_wide(ev[j], ev[j + 1], a.l[j], b0);
        mul_wide(od[j], od[j + 1], a.l[j + 1], b0);
    }
    mont_reduce_row(ev, od);
#pragma unroll
    for (int i = 1; i < 12; i += 2) {
        mont_mul_row(od, ev, a.l, b.l[i]);      // roles swap every row
        mont_reduce_row(od, ev);
        if (i + 1 < 12) {
            mont_mul_row(ev, od, a.l, b.l[i + 1]);
            mont_reduce_row(ev, od);
        }
    }
    // last row (i = 11) used E = od, O = ev:  T/2^32 = (od >> 32) + ev
    fp r;
    r.l[0] = add_cc(ev[0], od[1]);
#pragma unroll
    for (int k = 1; k < 11; k++) r.l[k] = addc_cc(ev[k], od[k + 1]);
    r.l[11] = addc(ev[11], 0);
    return r;
}
HD fp fp_mul(const fp& a, const fp& b) {
    fp r = fp_mul_lazy(a, b);
    fp_final_sub(r.l);
    return r;
}

// Dedicated squaring (separated operand scanning): 66 off-diagonal + 12 diagonal wide products for the 768-bit
// square, then a Montgomery reduction of the whole square in place (144 wide products) -- 222 IMAD.WIDE instead of
// the 288 of fp_mul(a, a).
//
// Off-diagonal terms a_i*a_j (i < j) land on limbs (s, s+1), s = i+j.  For a fixed i the terms with j = i+1, i+3, ...
// sit on consecutive ODD-aligned limb pairs and those with j = i+2, i+4, ... on consecutive EVEN-aligned pairs: each is
// one carry chain, into the accumulator of its alignment (uo / ue, indexed by absolute limb).  Rows are processed in
// increasing i; a chain's carry-out is absorbed by the limb just above it, which at that moment holds nothing but
// earlier absorbed carries (every product that lands there belongs to a later row), so it cannot overflow.

// 2N-limb square of an N-limb number (N even), separated operand scanning as described above: N(N-1)/2 + N wide products.
template <int N>
HD void sqr_limbs(const uint32_t* a, uint32_t* t) {
    uint32_t ue[2 * N], uo[2 * N];
#pragma unroll
    for (int k = 0; k < 2 * N; k++) ue[k] = uo[k] = 0u;
#pragma unroll
    for (int i = 0; i < N - 1; i++) {
        {   // j = i+1, i+3, ...  -> odd-aligned pairs
            mad_wide_cc(uo[2 * i + 1], uo[2 * i + 2], a[i], a[i + 1]);
            int s = 2 * i + 1;
#pragma unroll
            for (int j = i + 3; j < N; j += 2) {
                s = i + j;
                madc_wide_cc(uo[s], uo[s + 1], a[i], a[j]);
            }
            if (s + 2 < 2 * N) uo[s + 2] = addc(uo[s + 2], 0u);
        }
        if (i + 2 < N) {   // j = i+2, i+4, ...  -> even-aligned pairs
            mad_wide_cc(ue[2 * i + 2], ue[2 * i + 3], a[i], a[i + 2]);
            int s = 2 * i + 2;
#pragma unroll
            for (int j = i + 4; j < N; j += 2) {
                s = i + j;
                madc_wide_cc(ue[s], ue[s + 1], a[i], a[j]);
            }
            if (s + 2 < 2 * N) ue[s + 2] = addc(ue[s + 2], 0u);
        }
    }
    // t = 2*(ue + uo) + sum a_i^2 B^(2i)
    uint32_t d[2 * N];
    t[0] = add_cc(ue[0], uo[0]);
#pragma unroll
    for (int k = 1; k < 2 * N; k++) t[k] = addc_cc(ue[k], uo[k]);
    // doubling by funnel shifts (independent ops instead of a carry chain); the off-diagonal sum is < 2^(64N-1), nothing is shifted out
#pragma unroll
    for (int k = 2 * N - 1; k >= 1; k--) t[k] = (t[k] << 1) | (t[k - 1] >> 31);
    t[0] <<= 1;
#pragma unroll
    for (int i = 0; i < N; i++) mul_wide(d[2 * i], d[2 * i + 1], a[i], a[i]);
    t[0] = add_cc(t[0], d[0]);
#pragma unroll
    for (int k = 1; k < 2 * N - 1; k++) t[k] = addc_cc(t[k], d[k]);
    t[2 * N - 1] = addc(t[2 * N - 1], d[2 * N - 1]);
}

// 24-limb square of a 12-limb number.  B2_SQR_KARATSUBA selects one Karatsuba level over 6-limb halves a = a0 + a1*2^192:
//   a^2 = a0^2 + (a0^2 + a1^2 - (a0 - a1)^2) * 2^192 + a1^2 * 2^384
// i.e. three 6-limb squares (63 wide products) instead of 78.  Off: it measured slower (tools/pow_mix_bench.cu times
// both forms; not re-measured on the H100).  ptxas turns part of the extra carry
// bookkeeping into IMAD.X / IMAD.MOV (190 + 94 instead of 209 + 47 instructions on the FMA pipes per squaring), which costs more
// multiply-pipe time than the 19 wide products save.  Kept, tested by tests/test_hostsim.py, as the record of that experiment.
HD void sqr_product(const uint32_t* a, uint32_t* t) {
#if B2_SQR_KARATSUBA
    uint32_t dd[6], D[12], M[13];
    // dd = |a0 - a1|
    dd[0] = sub_cc(a[0], a[6]);
#pragma unroll
    for (int k = 1; k < 6; k++) dd[k] = subc_cc(a[k], a[6 + k]);
    const uint32_t neg = subc(0u, 0u);                      // all-ones when a0 < a1
    dd[0] = add_cc(dd[0] ^ neg, neg & 1u);
#pragma unroll
    for (int k = 1; k < 5; k++) dd[k] = addc_cc(dd[k] ^ neg, 0u);
    dd[5] = addc(dd[5] ^ neg, 0u);
    sqr_limbs<6>(a, t);                                     // L = a0^2 -> t[0..11]
    sqr_limbs<6>(a + 6, t + 12);                            // H = a1^2 -> t[12..23]
    sqr_limbs<6>(dd, D);
    // M = L + H - D = 2 a0 a1  (< 2^385: 13 limbs)
    M[0] = add_cc(t[0], t[12]);
#pragma unroll
    for (int k = 1; k < 12; k++) M[k] = addc_cc(t[k], t[12 + k]);
    M[12] = addc(0u, 0u);
    M[0] = sub_cc(M[0], D[0]);
#pragma unroll
    for (int k = 1; k < 12; k++) M[k] = subc_cc(M[k], D[k]);
    M[12] = subc(M[12], 0u);
    // t += M * 2^192
    t[6] = add_cc(t[6], M[0]);
#pragma unroll
    for (int k = 1; k < 13; k++) t[6 + k] = addc_cc(t[6 + k], M[k]);
#pragma unroll
    for (int k = 19; k < 23; k++) t[k] = addc_cc(t[k], 0u);
    t[23] = addc(t[23], 0u);
#else
    sqr_limbs<12>(a, t);
#endif
}

// Montgomery reduction of the 24-limb square in place (separated operand scanning, indexed by absolute limb): row i takes
// m = t[i]*(-p^-1) and adds m*p at limb i as the two alignment chains of mont_reduce_row, the even-j products onto the limb pairs
// that start at i's parity, the odd-j ones onto the pairs of the other parity.  Afterwards limb i is zero, so the division by
// 2^32 is only the next row starting one limb higher.  A 64-bit IMAD.WIDE operand is an aligned register pair, so each
// alignment keeps its own accumulator: A holds the pairs that start at even limbs, B those that start at odd limbs (one array
// for both would put every limb in a low and a high half within one row, and ptxas then spends a MOV per product).  Row i first
// folds limb i of the other accumulator into its own (the carry enters the odd-j chain, which starts at limb i+1).
// Carries: the even-j chain carries out at limb i+12, the odd-j chain at limb i+13, each into the LOW limb of a pair of its
// accumulator.  The high half of the square therefore sits on the HIGH limbs of the pairs only (odd limbs 13..23 in A, even
// limbs 12..22 in B), so a carry never lands on product data: before row i, limb i+12 of its accumulator holds at most the
// previous row's one-bit carry and limb i+13 nothing, and neither can overflow.
// Bound: for a < 2p, a^2 + M*p < 4p^2 + R*p with M < R; as p < R/8 that is < R * 1.5p < R^2, so the carry out of limb 23
// (last row) is zero, and (A + B)[12..23] = (a^2 + M*p)/R < 1.5p.  For a < p the result is < 1.125p.
HD fp fp_sqr_lazy(const fp& a) {
    uint32_t t[24], A[24], B[24];
    sqr_product(a.l, t);
#pragma unroll
    for (int k = 0; k < 24; k++) {
        const bool in_b = k >= 12 && !(k & 1);
        A[k] = in_b ? 0u : t[k];
        B[k] = in_b ? t[k] : 0u;
    }
#pragma unroll
    for (int i = 0; i < 12; i++) {
        uint32_t* X = (i & 1) ? B : A;          // pairs (i, i+1), (i+2, i+3), ...
        uint32_t* Y = (i & 1) ? A : B;          // pairs (i+1, i+2), ...
        if (i > 0) X[i] = add_cc(X[i], Y[i]);
        const uint32_t m = X[i] * B2_MONT_INV;
        if (i > 0) madc_wide_cc(Y[i + 1], Y[i + 2], P_LIMB(1), m);
        else mad_wide_cc(Y[i + 1], Y[i + 2], P_LIMB(1), m);
#pragma unroll
        for (int j = 3; j < 12; j += 2) madc_wide_cc(Y[i + j], Y[i + j + 1], P_LIMB(j), m);
        if (i + 13 < 24) Y[i + 13] = addc(Y[i + 13], 0u);
        mad_wide_cc(X[i], X[i + 1], P_LIMB(0), m);
#pragma unroll
        for (int j = 2; j < 12; j += 2) madc_wide_cc(X[i + j], X[i + j + 1], P_LIMB(j), m);
        X[i + 12] = addc(X[i + 12], 0u);
    }
    fp r;
    r.l[0] = add_cc(A[12], B[12]);
#pragma unroll
    for (int k = 1; k < 11; k++) r.l[k] = addc_cc(A[12 + k], B[12 + k]);
    r.l[11] = addc(A[23], B[23]);
    return r;
}
HD fp fp_sqr(const fp& a) {
    fp r = fp_sqr_lazy(a);
    fp_final_sub(r.l);
    return r;
}

// canonical <-> Montgomery
HD fp fp_to_mont(const fp& a) { return fp_mul(a, fp_load_const(C_R2)); }
HD fp fp_from_mont(const fp& a) {
    fp one = fp_zero();
    one.l[0] = 1;
    return fp_mul(a, one);
}

// small multiples
HD fp fp_mul3(const fp& a) { return fp_add(fp_dbl(a), a); }
HD fp fp_mul4(const fp& a) { return fp_dbl(fp_dbl(a)); }
HD fp fp_mul8(const fp& a) { return fp_dbl(fp_mul4(a)); }

// a^e for a fixed exponent given as a sliding-window schedule in the constant table (tools/gen_consts.py:
// word 0 = number of steps, then (n_squarings << 8 | table index), index 255 = squarings only; window 4, table of the
// eight odd powers a^1..a^15 plus a^255).  The schedule is the same in every thread, so nothing diverges.  For (p-3)/4 this is
// 380 squarings + 76 multiplications in all (375 + 68 in the schedule, 1 + 7 for the odd powers, 4 + 1 for a^255); the plain
// window-4 parse of round 1 needed 376 + 85, the fixed-window version 380 + 106.
// Where the eight odd powers live.  pow_tbl_local: a per-thread array -- dynamically indexed, so the compiler puts it in LOCAL memory
// (384 B per thread; with 16 resident warps per SM these tables overflow L1 and their evicted lines are what made k_g2_decompress
// write 1.2 GB to DRAM per launch, as measured on an earlier GPU).  A shared-memory form of the table (108 words per thread,
// conflict-free) was measured and dropped: it halved the decompression's DRAM traffic (1.40 -> 0.73 GB per launch), but its 48 KB
// per block competed with the tail kernels' shared memory under the epoch pipeline, and the step was 0.6 ms slower there (36.11 vs
// 35.48 ms, on an earlier GPU).
struct pow_tbl_local {
    fp t[9];
    HD void set(int i, const fp& v) { t[i] = v; }
    HD fp get(uint32_t i) const { return t[i]; }
};
// Inside the chain nothing is compared or encoded, so the table and every step stay in [0, 2p) (the lazy forms take and return
// values there); only the result is reduced.  `a` may itself lie anywhere in [0, 2p).
template <class TBL> HDN fp fp_pow_prog_t(const fp& a, int off, TBL& tbl) {
    const uint32_t* prog = const_table() + off;
    fp a2 = fp_sqr_lazy(a);
    fp cur = a;
    tbl.set(0, cur);
#pragma unroll 1
    for (int i = 1; i < 8; i++) {
        cur = fp_mul_lazy(cur, a2);
        tbl.set(i, cur);
    }
    // entry 8 = a^255 = (a^15)^16 * a^15: the run token of tools/gen_consts.py:token_program (one multiplication per EIGHT
    // consecutive one-bits of the exponent instead of one per four; (p-3)/4 has runs of 33, 19, 17, 10, 8 and 6)
    {
        fp t = cur;
#pragma unroll 1
        for (int i = 0; i < 4; i++) t = fp_sqr_lazy(t);
        tbl.set(8, fp_mul_lazy(t, cur));
    }
    const uint32_t n = prog[0];
    fp r = tbl.get(prog[1] & 0xffu);
#pragma unroll 1
    for (uint32_t k = 2; k <= n; k++) {
        const uint32_t op = prog[k];
#pragma unroll 1
        for (uint32_t s = op >> 8; s; s--) r = fp_sqr_lazy(r);
        const uint32_t idx = op & 0xffu;
        if (idx != 0xffu) r = fp_mul_lazy(r, tbl.get(idx));
    }
    fp_final_sub(r.l);
    return r;
}
HD fp fp_pow_prog(const fp& a, int off) {
    pow_tbl_local t;
    return fp_pow_prog_t(a, off, t);
}

HD fp fp_inv(const fp& a) { return fp_pow_prog(a, C_PROG_PM2); }        // 0 -> 0

// d = a^((p-3)/4).  Then a*d = a^((p+1)/4) is the square-root candidate and, when a is a
// non-zero square, d = 1/sqrt(a).
HD fp fp_pow_pm3d4(const fp& a) { return fp_pow_prog(a, C_PROG_PM3D4); }

// sqrt in Fp: returns true and writes a root when `a` is a square
HD bool fp_sqrt(const fp& a, fp& root) {
    fp d = fp_pow_pm3d4(a);
    root = fp_mul(d, a);
    return fp_eq(fp_sqr(root), a);
}

// "lexicographically largest" test on the canonical value: a > (p-1)/2
HD bool fp_is_lex_large_canonical(const fp& canon) {
    const uint32_t* h = const_table() + C_HALF_P;
    uint32_t t = sub_cc(h[0], canon.l[0]);
#pragma unroll
    for (int i = 1; i < 12; i++) t = subc_cc(h[i], canon.l[i]);
    (void)t;
    return subc(0, 0) != 0;                     // borrow <=> half_p < a
}

// big-endian 48-byte encoding <-> canonical limbs
HD void fp_to_be48(const fp& canon, uint8_t* out) {
#pragma unroll
    for (int i = 0; i < 12; i++) {
        uint32_t w = canon.l[11 - i];
        out[4 * i + 0] = (uint8_t)(w >> 24);
        out[4 * i + 1] = (uint8_t)(w >> 16);
        out[4 * i + 2] = (uint8_t)(w >> 8);
        out[4 * i + 3] = (uint8_t)w;
    }
}
// the same from twelve 32-bit words loaded as they lie in memory (little-endian loads of big-endian bytes): one byte swap per limb
HD fp fp_from_be48_words(const uint32_t* w) {
    fp r;
#pragma unroll
    for (int i = 0; i < 12; i++) {
        const uint32_t v = w[i];
        r.l[11 - i] = (v >> 24) | ((v >> 8) & 0xff00u) | ((v << 8) & 0xff0000u) | (v << 24);
    }
    return r;
}
HD fp fp_from_be48(const uint8_t* in) {
    fp r;
#pragma unroll
    for (int i = 0; i < 12; i++)
        r.l[11 - i] = ((uint32_t)in[4 * i] << 24) | ((uint32_t)in[4 * i + 1] << 16) | ((uint32_t)in[4 * i + 2] << 8) | in[4 * i + 3];
    return r;
}
// canonical value < p ?
HD bool fp_canonical_lt_p(const fp& canon) {
    uint32_t t = sub_cc(canon.l[0], P_LIMB(0));
#pragma unroll
    for (int i = 1; i < 12; i++) t = subc_cc(canon.l[i], P_LIMB(i));
    (void)t;
    return subc(0, 0) != 0;
}

}  // namespace b2
