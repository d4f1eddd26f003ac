// fp2.cuh -- Fp2 = Fp[i]/(i^2+1); element c0 + c1*i.  Part of kernel library K1 (SURVEY.md section 2).
#pragma once
#include "fp.cuh"

namespace b2 {

struct fp2 {
    fp c0, c1;
};

HD fp2 fp2_load_const(int off) {
    fp2 r;
    r.c0 = fp_load_const(off);
    r.c1 = fp_load_const(off + 12);
    return r;
}
HD fp2 fp2_zero() {
    fp2 r;
    r.c0 = fp_zero();
    r.c1 = fp_zero();
    return r;
}
HD fp2 fp2_one() {
    fp2 r;
    r.c0 = fp_one();
    r.c1 = fp_zero();
    return r;
}
HD fp2 fp2_from_fp(const fp& a) {
    fp2 r;
    r.c0 = a;
    r.c1 = fp_zero();
    return r;
}
HD bool fp2_is_zero(const fp2& a) { return fp_is_zero(a.c0) && fp_is_zero(a.c1); }
HD bool fp2_eq(const fp2& a, const fp2& b) { return fp_eq(a.c0, b.c0) && fp_eq(a.c1, b.c1); }
HD fp2 fp2_select(bool c, const fp2& a, const fp2& b) {
    fp2 r;
    r.c0 = fp_select(c, a.c0, b.c0);
    r.c1 = fp_select(c, a.c1, b.c1);
    return r;
}
HD fp2 fp2_add(const fp2& a, const fp2& b) {
    fp2 r;
    r.c0 = fp_add(a.c0, b.c0);
    r.c1 = fp_add(a.c1, b.c1);
    return r;
}
HD fp2 fp2_sub(const fp2& a, const fp2& b) {
    fp2 r;
    r.c0 = fp_sub(a.c0, b.c0);
    r.c1 = fp_sub(a.c1, b.c1);
    return r;
}
HD fp2 fp2_neg(const fp2& a) {
    fp2 r;
    r.c0 = fp_neg(a.c0);
    r.c1 = fp_neg(a.c1);
    return r;
}
HD fp2 fp2_dbl(const fp2& a) { return fp2_add(a, a); }
HD fp2 fp2_conj(const fp2& a) {
    fp2 r;
    r.c0 = a.c0;
    r.c1 = fp_neg(a.c1);
    return r;
}
// Karatsuba: 3 Fp multiplications
HDN fp2 fp2_mul(const fp2& a, const fp2& b) {
    fp t0 = fp_mul(a.c0, b.c0);
    fp t1 = fp_mul(a.c1, b.c1);
    fp s = fp_mul(fp_add(a.c0, a.c1), fp_add(b.c0, b.c1));
    fp2 r;
    r.c0 = fp_sub(t0, t1);
    r.c1 = fp_sub(fp_sub(s, t0), t1);
    return r;
}
// (a0+a1)(a0-a1) + 2*a0*a1*i : 2 Fp multiplications
HDN fp2 fp2_sqr(const fp2& a) {
    fp t = fp_mul(a.c0, a.c1);
    fp2 r;
    r.c0 = fp_mul(fp_add(a.c0, a.c1), fp_sub(a.c0, a.c1));
    r.c1 = fp_dbl(t);
    return r;
}
HDN fp2 fp2_mul_fp(const fp2& a, const fp& k) {
    fp2 r;
    r.c0 = fp_mul(a.c0, k);
    r.c1 = fp_mul(a.c1, k);
    return r;
}
// multiply by xi = 1 + i
HD fp2 fp2_mul_xi(const fp2& a) {
    fp2 r;
    r.c0 = fp_sub(a.c0, a.c1);
    r.c1 = fp_add(a.c0, a.c1);
    return r;
}
HD fp2 fp2_mul3(const fp2& a) { return fp2_add(fp2_dbl(a), a); }
HD fp2 fp2_mul4(const fp2& a) { return fp2_dbl(fp2_dbl(a)); }
HD fp2 fp2_mul8(const fp2& a) { return fp2_dbl(fp2_mul4(a)); }

HDN fp2 fp2_inv(const fp2& a) {
    fp n = fp_add(fp_sqr(a.c0), fp_sqr(a.c1));
    fp d = fp_inv(n);
    fp2 r;
    r.c0 = fp_mul(a.c0, d);
    r.c1 = fp_neg(fp_mul(a.c1, d));
    return r;
}

// Square root in Fp2 with exactly two Fp exponentiations (p = 3 mod 4, "complex method"):
//   n = a0^2 + a1^2 must be a square s^2 in Fp;  t = (a0 + s)/2;  d = t^((p-3)/4), x = d*t.
//   If x^2 == t:  root = x + (a1*d/2) i          (d = 1/x)
//   else       :  root = (a1*d/2) - x i          (d^2 = -1/t, so (a1*d/2)^2 = (a0 - s)/2)
// Returns false when `a` is not a square.  Any root; callers fix the sign.
HDN bool fp2_sqrt(const fp2& a, fp2& r) {
    if (fp_is_zero(a.c1)) {                      // a in Fp: always a square in Fp2
        fp x;
        bool qr = fp_sqrt(a.c0, x);              // x = a0^((p+1)/4); x^2 = -a0 when a0 is a non-residue
        r.c0 = qr ? x : fp_zero();
        r.c1 = qr ? fp_zero() : x;
        return true;
    }
    fp n = fp_add(fp_sqr(a.c0), fp_sqr(a.c1));
    fp s = fp_mul(fp_pow_pm3d4(n), n);
    if (!fp_eq(fp_sqr(s), n)) return false;
    fp half = fp_load_const(C_TWO_INV);
    fp t = fp_mul(fp_add(a.c0, s), half);
    fp d = fp_pow_pm3d4(t);
    fp x = fp_mul(d, t);
    fp y = fp_mul(fp_mul(a.c1, half), d);
    bool direct = fp_eq(fp_sqr(x), t);
    r.c0 = fp_select(direct, x, y);
    r.c1 = fp_select(direct, y, fp_neg(x));
    return true;
}

// RFC 9380 sgn0 for m = 2 (needs canonical values)
HD uint32_t fp2_sgn0(const fp2& a) {
    fp c0 = fp_from_mont(a.c0), c1 = fp_from_mont(a.c1);
    uint32_t s0 = c0.l[0] & 1u;
    uint32_t z0 = fp_is_zero(c0) ? 1u : 0u;
    uint32_t s1 = c1.l[0] & 1u;
    return s0 | (z0 & s1);
}

// ZCash "lexicographically largest": compare c1 first, then c0 (canonical values)
HD bool fp2_is_lex_large(const fp2& a) {
    fp c1 = fp_from_mont(a.c1);
    if (!fp_is_zero(c1)) return fp_is_lex_large_canonical(c1);
    return fp_is_lex_large_canonical(fp_from_mont(a.c0));
}

}  // namespace b2
