// curve.cuh -- E1: y^2 = x^3 + 4 over Fp and E2: y^2 = x^3 + 4(1+i) over Fp2, Jacobian coordinates
// (x = X/Z^2, y = Y/Z^3, infinity <=> Z == 0), ZCash point encodings, subgroup checks.
// One template serves both groups.  This is the arithmetic behind kernels K2 (G1 pubkey
// aggregation) and K3 (G2 signature aggregation) of SURVEY.md section 2; the reference reaches it only
// through bls.* call sites (pos-evolution.md:165, :736, :976).
#pragma once
#include "fp2.cuh"

namespace b2 {

// ---- field-generic names
HD fp f_add(const fp& a, const fp& b) { return fp_add(a, b); }
HD fp f_sub(const fp& a, const fp& b) { return fp_sub(a, b); }
HD fp f_mul(const fp& a, const fp& b) { return fp_mul(a, b); }
HD fp f_sqr(const fp& a) { return fp_sqr(a); }
HD fp f_neg(const fp& a) { return fp_neg(a); }
HD fp f_dbl(const fp& a) { return fp_dbl(a); }
HD fp f_inv(const fp& a) { return fp_inv(a); }
HD bool f_is_zero(const fp& a) { return fp_is_zero(a); }
HD bool f_eq(const fp& a, const fp& b) { return fp_eq(a, b); }
HD fp f_select(bool c, const fp& a, const fp& b) { return fp_select(c, a, b); }
HD fp2 f_add(const fp2& a, const fp2& b) { return fp2_add(a, b); }
HD fp2 f_sub(const fp2& a, const fp2& b) { return fp2_sub(a, b); }
HD fp2 f_mul(const fp2& a, const fp2& b) { return fp2_mul(a, b); }
HD fp2 f_sqr(const fp2& a) { return fp2_sqr(a); }
HD fp2 f_neg(const fp2& a) { return fp2_neg(a); }
HD fp2 f_dbl(const fp2& a) { return fp2_dbl(a); }
HD fp2 f_inv(const fp2& a) { return fp2_inv(a); }
HD bool f_is_zero(const fp2& a) { return fp2_is_zero(a); }
HD bool f_eq(const fp2& a, const fp2& b) { return fp2_eq(a, b); }
HD fp2 f_select(bool c, const fp2& a, const fp2& b) { return fp2_select(c, a, b); }
template <class F> HD F f_zero();
template <> HD fp f_zero<fp>() { return fp_zero(); }
template <> HD fp2 f_zero<fp2>() { return fp2_zero(); }
template <class F> HD F f_one();
template <> HD fp f_one<fp>() { return fp_one(); }
template <> HD fp2 f_one<fp2>() { return fp2_one(); }
template <class F> HD F curve_b();
template <> HD fp curve_b<fp>() { return fp_load_const(C_FOUR); }
template <> HD fp2 curve_b<fp2>() { return fp2_load_const(C_B2); }

template <class F> struct jac {
    F x, y, z;
};
template <class F> struct aff {
    F x, y;
};
typedef jac<fp> g1_jac;
typedef aff<fp> g1_aff;
typedef jac<fp2> g2_jac;
typedef aff<fp2> g2_aff;

template <class F> HD jac<F> pt_inf() {
    jac<F> r;
    r.x = f_one<F>();
    r.y = f_one<F>();
    r.z = f_zero<F>();
    return r;
}
template <class F> HD bool pt_is_inf(const jac<F>& p) { return f_is_zero(p.z); }
template <class F> HD jac<F> pt_from_affine(const aff<F>& a) {
    jac<F> r;
    r.x = a.x;
    r.y = a.y;
    r.z = f_one<F>();
    return r;
}
template <class F> HD jac<F> pt_neg(const jac<F>& p) {
    jac<F> r = p;
    r.y = f_neg(p.y);
    return r;
}
template <class F> HD jac<F> pt_select(bool c, const jac<F>& a, const jac<F>& b) {
    jac<F> r;
    r.x = f_select(c, a.x, b.x);
    r.y = f_select(c, a.y, b.y);
    r.z = f_select(c, a.z, b.z);
    return r;
}
template <class F> HD bool aff_on_curve(const aff<F>& a) {
    return f_eq(f_sqr(a.y), f_add(f_mul(f_sqr(a.x), a.x), curve_b<F>()));
}

// dbl-2009-l (a = 0): 2M + 5S.  Z = 0 stays Z = 0.
template <class F> HDN jac<F> pt_dbl(const jac<F>& p) {
    F A = f_sqr(p.x);
    F B = f_sqr(p.y);
    F C = f_sqr(B);
    F D = f_dbl(f_sub(f_sub(f_sqr(f_add(p.x, B)), A), C));
    F E = f_add(f_dbl(A), A);
    F Fq = f_sqr(E);
    jac<F> r;
    r.x = f_sub(Fq, f_dbl(D));
    F C8 = f_dbl(f_dbl(f_dbl(C)));
    r.y = f_sub(f_mul(E, f_sub(D, r.x)), C8);
    r.z = f_dbl(f_mul(p.y, p.z));
    return r;
}

// madd-2007-bl: Jacobian + affine, 7M + 4S, all exceptional cases handled (rare branches)
template <class F> HDN jac<F> pt_add_mixed(const jac<F>& p, const aff<F>& q) {
    if (pt_is_inf(p)) return pt_from_affine(q);
    F Z1Z1 = f_sqr(p.z);
    F U2 = f_mul(q.x, Z1Z1);
    F S2 = f_mul(f_mul(q.y, p.z), Z1Z1);
    F H = f_sub(U2, p.x);
    F rr = f_sub(S2, p.y);
    if (f_is_zero(H)) {
        if (f_is_zero(rr)) return pt_dbl(p);
        return pt_inf<F>();
    }
    rr = f_dbl(rr);
    F HH = f_sqr(H);
    F I = f_dbl(f_dbl(HH));
    F J = f_mul(H, I);
    F V = f_mul(p.x, I);
    jac<F> r;
    r.x = f_sub(f_sub(f_sqr(rr), J), f_dbl(V));
    r.y = f_sub(f_mul(rr, f_sub(V, r.x)), f_dbl(f_mul(p.y, J)));
    r.z = f_sub(f_sub(f_sqr(f_add(p.z, H)), Z1Z1), HH);
    return r;
}

// add-2007-bl: Jacobian + Jacobian, 11M + 5S
template <class F> HDN jac<F> pt_add(const jac<F>& p, const jac<F>& q) {
    if (pt_is_inf(p)) return q;
    if (pt_is_inf(q)) return p;
    F Z1Z1 = f_sqr(p.z);
    F Z2Z2 = f_sqr(q.z);
    F U1 = f_mul(p.x, Z2Z2);
    F U2 = f_mul(q.x, Z1Z1);
    F S1 = f_mul(f_mul(p.y, q.z), Z2Z2);
    F S2 = f_mul(f_mul(q.y, p.z), Z1Z1);
    F H = f_sub(U2, U1);
    F rr = f_sub(S2, S1);
    if (f_is_zero(H)) {
        if (f_is_zero(rr)) return pt_dbl(p);
        return pt_inf<F>();
    }
    rr = f_dbl(rr);
    F I = f_sqr(f_dbl(H));
    F J = f_mul(H, I);
    F V = f_mul(U1, I);
    jac<F> r;
    r.x = f_sub(f_sub(f_sqr(rr), J), f_dbl(V));
    r.y = f_sub(f_mul(rr, f_sub(V, r.x)), f_dbl(f_mul(S1, J)));
    r.z = f_mul(f_sub(f_sub(f_sqr(f_add(p.z, q.z)), Z1Z1), Z2Z2), H);
    return r;
}

template <class F> HDN bool pt_eq(const jac<F>& p, const jac<F>& q) {
    bool pi = pt_is_inf(p), qi = pt_is_inf(q);
    if (pi || qi) return pi && qi;
    F Z1Z1 = f_sqr(p.z), Z2Z2 = f_sqr(q.z);
    if (!f_eq(f_mul(p.x, Z2Z2), f_mul(q.x, Z1Z1))) return false;
    return f_eq(f_mul(f_mul(p.y, q.z), Z2Z2), f_mul(f_mul(q.y, p.z), Z1Z1));
}

// -> affine; returns false for infinity (out untouched)
template <class F> HDN bool pt_to_affine(const jac<F>& p, aff<F>& out) {
    if (pt_is_inf(p)) return false;
    F zi = f_inv(p.z);
    F zi2 = f_sqr(zi);
    out.x = f_mul(p.x, zi2);
    out.y = f_mul(p.y, f_mul(zi2, zi));
    return true;
}

// [k]P for a scalar that is the same in every thread (loop-uniform branches): 64-bit k
template <class F> HDN jac<F> pt_mul_u64(const jac<F>& p, uint64_t k) {
    jac<F> r = pt_inf<F>();
    bool started = false;
#pragma unroll 1
    for (int i = 63; i >= 0; i--) {
        if (started) r = pt_dbl(r);
        if ((k >> i) & 1) {
            r = started ? pt_add(r, p) : p;
            started = true;
        }
    }
    return r;
}
// [k]P, k = `nlimbs` 32-bit limbs in the constant table (uniform)
template <class F> HDN jac<F> pt_mul_const(const jac<F>& p, int off, int nlimbs) {
    const uint32_t* e = const_table() + off;
    jac<F> r = pt_inf<F>();
    bool started = false;
#pragma unroll 1
    for (int i = nlimbs * 32 - 1; i >= 0; i--) {
        if (started) r = pt_dbl(r);
        if ((e[i >> 5] >> (i & 31)) & 1u) {
            r = started ? pt_add(r, p) : p;
            started = true;
        }
    }
    return r;
}
// [k]P for a per-thread scalar (8 x 32-bit limbs, little endian): branch-free double-and-always-add
template <class F> HDN jac<F> pt_mul_var(const jac<F>& p, const uint32_t* k) {
    jac<F> r = pt_inf<F>();
#pragma unroll 1
    for (int i = 255; i >= 0; i--) {
        r = pt_dbl(r);
        jac<F> s = pt_add(r, p);
        r = pt_select(((k[i >> 5] >> (i & 31)) & 1u) != 0, s, r);
    }
    return r;
}

// ------------------------------------------------------------------------------------------ ZCash encodings
enum DecodeStatus : int { DEC_OK = 0, DEC_INF = 1, DEC_BAD = 2 };

// 48 bytes -> affine G1 point (Montgomery coordinates).  On-curve is implied; subgroup NOT checked.
HDN int g1_decompress(const uint8_t* in, g1_aff& out) {
    uint8_t b0 = in[0];
    if (!(b0 & 0x80)) return DEC_BAD;
    fp xc = fp_from_be48(in);
    xc.l[11] &= 0x1fffffffu;
    if (b0 & 0x40) {
        if ((b0 & 0x20) || !fp_is_zero(xc)) return DEC_BAD;
        return DEC_INF;
    }
    if (!fp_canonical_lt_p(xc)) return DEC_BAD;
    fp x = fp_to_mont(xc);
    fp y;
    if (!fp_sqrt(fp_add(fp_mul(fp_sqr(x), x), fp_load_const(C_FOUR)), y)) return DEC_BAD;
    bool large = fp_is_lex_large_canonical(fp_from_mont(y));
    if (large != ((b0 & 0x20) != 0)) y = fp_neg(y);
    out.x = x;
    out.y = y;
    return DEC_OK;
}
HDN void g1_compress_affine(const g1_aff& a, bool inf, uint8_t* out) {
    if (inf) {
#pragma unroll 1
        for (int i = 0; i < 48; i++) out[i] = 0;
        out[0] = 0xC0;
        return;
    }
    fp_to_be48(fp_from_mont(a.x), out);
    out[0] |= 0x80 | (fp_is_lex_large_canonical(fp_from_mont(a.y)) ? 0x20 : 0);
}
HD void g1_compress(const g1_jac& p, uint8_t* out) {
    g1_aff a;
    a.x = fp_zero();
    a.y = fp_zero();
    bool ok = pt_to_affine(p, a);
    g1_compress_affine(a, !ok, out);
}

// 96 bytes (x.c1 || x.c0) -> affine G2 point.  On-curve implied; subgroup NOT checked.
HDN int g2_decompress(const uint8_t* in, g2_aff& out) {
    fp x1c, x0c;
    uint8_t b0;
#if defined(__CUDA_ARCH__) && defined(B2_SIG_VECTOR_LOADS)
    {
        // 96 contiguous bytes per signature as six 128-bit loads (needs 16-byte aligned signature arrays).  MEASURED SLOWER than the
        // byte loads below and therefore off: 29.47 vs 29.23 ms for 2^20 decompressions, twice, tools/decompress_bench.cu
        // (tools/decompress_bench.cu, on an earlier GPU).  The loads are 0.04 % of the kernel's instructions either way; the 24 live
        // words at the top of the function cost the register allocation of what follows more than the 90 saved LDG.U8 return.
        const uint4* in4 = reinterpret_cast<const uint4*>(in);
        const uint4 q0 = in4[0], q1 = in4[1], q2 = in4[2], q3 = in4[3], q4 = in4[4], q5 = in4[5];
        const uint32_t w1[12] = {q0.x, q0.y, q0.z, q0.w, q1.x, q1.y, q1.z, q1.w, q2.x, q2.y, q2.z, q2.w};
        const uint32_t w0[12] = {q3.x, q3.y, q3.z, q3.w, q4.x, q4.y, q4.z, q4.w, q5.x, q5.y, q5.z, q5.w};
        b0 = (uint8_t)(q0.x & 0xffu);
        x1c = fp_from_be48_words(w1);
        x0c = fp_from_be48_words(w0);
    }
#else
    {
        b0 = in[0];
        x1c = fp_from_be48(in);
        x0c = fp_from_be48(in + 48);
    }
#endif
    if (!(b0 & 0x80)) return DEC_BAD;
    x1c.l[11] &= 0x1fffffffu;
    if (b0 & 0x40) {
        if ((b0 & 0x20) || !fp_is_zero(x1c) || !fp_is_zero(x0c)) return DEC_BAD;
        return DEC_INF;
    }
    if (!fp_canonical_lt_p(x1c) || !fp_canonical_lt_p(x0c)) return DEC_BAD;
    fp2 x;
    x.c0 = fp_to_mont(x0c);
    x.c1 = fp_to_mont(x1c);
    fp2 y;
    if (!fp2_sqrt(fp2_add(fp2_mul(fp2_sqr(x), x), fp2_load_const(C_B2)), y)) return DEC_BAD;
    if (fp2_is_lex_large(y) != ((b0 & 0x20) != 0)) y = fp2_neg(y);
    out.x = x;
    out.y = y;
    return DEC_OK;
}
HDN void g2_compress_affine(const g2_aff& a, bool inf, uint8_t* out) {
    if (inf) {
#pragma unroll 1
        for (int i = 0; i < 96; i++) out[i] = 0;
        out[0] = 0xC0;
        return;
    }
    fp_to_be48(fp_from_mont(a.x.c1), out);
    fp_to_be48(fp_from_mont(a.x.c0), out + 48);
    out[0] |= 0x80 | (fp2_is_lex_large(a.y) ? 0x20 : 0);
}
HD void g2_compress(const g2_jac& p, uint8_t* out) {
    g2_aff a;
    a.x = fp2_zero();
    a.y = fp2_zero();
    bool ok = pt_to_affine(p, a);
    g2_compress_affine(a, !ok, out);
}

// ------------------------------------------------------------------------------------------ subgroup membership
// exact: [r]P == O  (used for KeyValidate at registry load, a one-time cost per validator)
template <class F> HD bool pt_in_subgroup_exact(const jac<F>& p) { return pt_is_inf(pt_mul_const(p, C_R_ORDER, 8)); }

// psi: untwist-Frobenius-twist endomorphism of E2 (RFC 9380 appendix G.3)
HD g2_jac g2_psi(const g2_jac& p) {
    g2_jac r;
    r.x = fp2_mul(fp2_conj(p.x), fp2_load_const(C_PSI_CX));
    r.y = fp2_mul(fp2_conj(p.y), fp2_load_const(C_PSI_CY));
    r.z = fp2_conj(p.z);
    return r;
}
HD g2_jac g2_psi2(const g2_jac& p) {
    g2_jac r;
    r.x = fp2_mul_fp(p.x, fp_load_const(C_PSI2_CX));
    r.y = fp2_neg(p.y);
    r.z = p.z;
    return r;
}
// Scott 2021 ("A note on group membership tests for G1, G2 and GT on BLS pairing-friendly curves"):
// P in G2  <=>  psi(P) == [x]P.  x = -|x|.  Equivalent to the oracle's [r]P == O (tests/test_hostsim.py
// checks both directions on subgroup and non-subgroup points).
HDN bool g2_in_subgroup(const g2_jac& p) {
    if (pt_is_inf(p)) return true;
    g2_jac xp = pt_neg(pt_mul_u64(p, B2_X_ABS));
    return pt_eq(g2_psi(p), xp);
}

}  // namespace b2
