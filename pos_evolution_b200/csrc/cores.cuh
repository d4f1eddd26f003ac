// cores.cuh -- per-thread bodies ("cores") of the BLS kernels, written as host+device code so
// that tests/hostsim can run exactly these bodies on the CPU against the oracle.  kernels.cu
// wraps them in __global__ functions and adds the warp/block-level reductions.
//
// Device-resident data formats (DESIGN.md "HBM layout"):
//   registry record   24 x u32   affine G1 pubkey (x, y), Montgomery limbs        96 B / validator
//   registry valid    u8         1 = KeyValidate passed (decodable, not infinity, in G1)
//   aggregated pubkey 36 x u32   Jacobian G1 (X, Y, Z), Montgomery                144 B / aggregate
//   G2 affine point   48 x u32   (x.c0, x.c1, y.c0, y.c1), Montgomery             192 B
//   Miller value      144 x u32  Fp12, tower order, Montgomery                    576 B
#pragma once
#include "h2c.cuh"
#include "pairing.cuh"

namespace b2 {

// status bits of an aggregated pubkey (mirrors the ways py_ecc FastAggregateVerify returns False)
enum PkStatus : uint32_t { PK_OK = 0, PK_INVALID_KEY = 1, PK_EMPTY = 2, PK_INFINITY = 4, PK_BAD_INDEX = 8 /* member index outside the registry, or a malformed committee row */ };
// signature flags
enum SigFlag : uint8_t { SIG_OK = 0, SIG_INFINITY = 1, SIG_INVALID = 2 };

HD uint8_t dst_pop_byte(int i) {
    constexpr char d[44] = "BLS_SIG_BLS12381G2_XMD:SHA-256_SSWU_RO_POP_";
    return (uint8_t)d[i];
}
#define B2_DST_POP_LEN 43

// ---- registry: decompress + KeyValidate one pubkey (done once per validator set, not per epoch)
HD void core_registry_load(const uint8_t* pk48, uint32_t* records, uint8_t* valid, uint64_t i) {
    g1_aff a;
    a.x = fp_zero();
    a.y = fp_zero();
    int s = g1_decompress(pk48 + 48 * i, a);
    bool ok = (s == DEC_OK) && pt_in_subgroup_exact(pt_from_affine(a));
    if (!ok) {
        a.x = fp_zero();
        a.y = fp_zero();
    }
    uint32_t* r = records + 24 * i;
#pragma unroll
    for (int k = 0; k < 12; k++) {
        r[k] = a.x.l[k];
        r[12 + k] = a.y.l[k];
    }
    valid[i] = ok ? 1 : 0;
}

HD g1_aff load_record(const uint32_t* records, uint32_t idx) {
    g1_aff a;
    const uint32_t* r = records + 24 * (uint64_t)idx;
#pragma unroll
    for (int k = 0; k < 12; k++) {
        a.x.l[k] = r[k];
        a.y.l[k] = r[12 + k];
    }
    return a;
}

// ---- K2: one member of one aggregate (bit j of aggregate a)
HD void core_g1_accumulate(const uint32_t* records, const uint8_t* valid, const uint32_t* members, const uint32_t* off,
                           const uint8_t* bits, uint32_t bits_stride, uint32_t a, uint32_t j, g1_jac& acc, uint32_t& status,
                           uint32_t& cnt, uint64_t n_val = ~0ull) {
    if (!((bits[(uint64_t)a * bits_stride + (j >> 3)] >> (j & 7)) & 1)) return;
    uint32_t idx = members[off[a] + j];
    cnt++;
    if (idx >= n_val) {                      // device-pointer entry points cannot be validated on the host: never read out of bounds
        status |= PK_BAD_INDEX;
        return;
    }
    if (!valid[idx]) {
        status |= PK_INVALID_KEY;
        return;
    }
    acc = pt_add_mixed(acc, load_record(records, idx));
}
HD void store_g1_jac(uint32_t* out, const g1_jac& p) {
#pragma unroll
    for (int k = 0; k < 12; k++) {
        out[k] = p.x.l[k];
        out[12 + k] = p.y.l[k];
        out[24 + k] = p.z.l[k];
    }
}
HD g1_jac load_g1_jac(const uint32_t* in) {
    g1_jac p;
#pragma unroll
    for (int k = 0; k < 12; k++) {
        p.x.l[k] = in[k];
        p.y.l[k] = in[12 + k];
        p.z.l[k] = in[24 + k];
    }
    return p;
}
HD void core_g1_finish(const g1_jac& acc, uint32_t status, uint32_t cnt, uint32_t a, uint32_t* out_jac, uint8_t* out_status) {
    if (cnt == 0) status |= PK_EMPTY;
    if (pt_is_inf(acc)) status |= PK_INFINITY;
    store_g1_jac(out_jac + 36 * (uint64_t)a, acc);
    out_status[a] = (uint8_t)status;
}

// ---- K3: one signature of a segment
HD void core_g2_accumulate(const uint8_t* sig96, uint64_t j, g2_jac& acc, uint32_t& bad) {
    g2_aff s;
    int st = g2_decompress(sig96 + 96 * j, s);
    if (st == DEC_BAD) {
        bad = 1;
        return;
    }
    if (st == DEC_INF) return;
    acc = pt_add_mixed(acc, s);
}
// seg_status: 0 ok, 1 undecodable signature in the segment (py_ecc raises), 2 empty segment (raises)
HD void core_g2_agg_finish(const g2_jac& acc, uint32_t bad, uint32_t count, uint32_t s, uint8_t* out96, int32_t* seg_status) {
    int32_t st = bad ? 1 : (count == 0 ? 2 : 0);
    seg_status[s] = st;
    if (st == 0) {
        g2_compress(acc, out96 + 96 * (uint64_t)s);
    } else {
#pragma unroll 1
        for (int k = 0; k < 96; k++) out96[96 * (uint64_t)s + k] = 0;
    }
}

// ---- K4: H(m) for aggregate a, affine
HD void core_hash_msg(const uint8_t* msg32, uint32_t a, g2_aff& h, uint8_t& hflag) {
    uint8_t dst[B2_DST_POP_LEN];
#pragma unroll 1
    for (int i = 0; i < B2_DST_POP_LEN; i++) dst[i] = dst_pop_byte(i);
    g2_jac q = hash_to_g2(msg32 + 32 * (uint64_t)a, 32, dst, B2_DST_POP_LEN);
    h.x = fp2_zero();
    h.y = fp2_zero();
    hflag = pt_to_affine(q, h) ? 0 : 1;
}
// ---- signature: decompress + subgroup check
HD void core_sig_prepare(const uint8_t* sig96, uint32_t a, g2_aff& s, uint8_t& sflag) {
    s.x = fp2_zero();
    s.y = fp2_zero();
    int st = g2_decompress(sig96 + 96 * (uint64_t)a, s);
    if (st == DEC_BAD) {
        sflag = SIG_INVALID;
    } else if (st == DEC_INF) {
        sflag = SIG_INFINITY;
    } else {
        sflag = g2_in_subgroup(pt_from_affine(s)) ? SIG_OK : SIG_INVALID;
    }
}
// ---- K5: the two Miller loops of  e(PK_agg, H(m)) * e(-g1, sig)
HD fp12 core_miller_pk(const uint32_t* pk_jac, const uint8_t* pk_status, uint32_t a, const g2_aff& h, uint8_t hflag) {
    if (pk_status[a] != PK_OK) return fp12_one();
    return miller_loop(load_g1_jac(pk_jac + 36 * (uint64_t)a), h, hflag != 0);
}
HD fp12 core_miller_sig(const g2_aff& s, uint8_t sflag) {
    if (sflag == SIG_INVALID) return fp12_one();
    g1_jac ng;
    ng.x = fp_load_const(C_G1X);
    ng.y = fp_load_const(C_G1Y_NEG);
    ng.z = fp_one();
    return miller_loop(ng, s, sflag == SIG_INFINITY);
}
// ---- K6: final exponentiation and verdict
HD uint8_t core_final_verdict(const fp12& f0, const fp12& f1, uint8_t pk_status, uint8_t sflag) {
    if (pk_status != PK_OK || sflag == SIG_INVALID) return 0;
    return fp12_is_one(final_exponentiation(fp12_mul(f0, f1))) ? 1 : 0;
}

// ---- bls.AggregateVerify, batched (kernels in aggverify.cuh).  Set s owns the items [pair_off[s] + s, pair_off[s+1] + s + 1): one per
// (key, message) pair, then one for its signature.  Every item is one Miller loop; the set's product of them takes ONE final
// exponentiation:  prod_i e(pk_i, H(m_i)) * e(-g1, S) == 1.  An item also yields the status bits that reject its set outright.
enum AvStatus : uint32_t { AV_BAD_KEY = 1, AV_BAD_INDEX = 2 /* signer index outside the registry */, AV_BAD_SIG = 4 };
// the set of item i: the last s whose first item pair_off[s] + s is <= i (first items strictly increase when pair_off is monotone)
HD uint32_t av_set_of(const uint32_t* pair_off, uint32_t n_sets, uint32_t i) {
    uint32_t lo = 0, hi = n_sets - 1;
#pragma unroll 1
    while (lo < hi) {
        const uint32_t mid = lo + (hi - lo + 1) / 2;
        if (pair_off[mid] + mid <= i) {
            lo = mid;
        } else {
            hi = mid - 1;
        }
    }
    return lo;
}
// The Miller-loop arguments of an item, so that pair and signature items of one warp share ONE call of miller_loop.
// Pair item: (pk, H(m)) with pk = key record idx of a table of n_keys; an index outside the table or a key that failed KeyValidate
// rejects the set and leaves P at infinity (the loop then returns 1 at once).
HD void core_av_pair(const uint32_t* records, const uint8_t* valid, uint32_t idx, uint64_t n_keys, const g2_aff& h, uint8_t hflag, g1_jac& p,
                     g2_aff& q, bool& q_inf, uint32_t& bad) {
    q = h;
    q_inf = hflag != 0;
    p = pt_inf<fp>();
    if (idx >= n_keys) {
        bad |= AV_BAD_INDEX;
    } else if (!valid[idx]) {
        bad |= AV_BAD_KEY;
    } else {
        p = pt_from_affine(load_record(records, idx));
    }
}
// Signature item: (-g1, S); an undecodable or non-G2 signature rejects the set
HD void core_av_sig(const g2_aff& s, uint8_t sflag, g1_jac& p, g2_aff& q, bool& q_inf, uint32_t& bad) {
    p.x = fp_load_const(C_G1X);
    p.y = fp_load_const(C_G1Y_NEG);
    p.z = fp_one();
    q = s;
    q_inf = sflag != SIG_OK;
    if (sflag == SIG_INVALID) bad |= AV_BAD_SIG;
}
// F = the product of the set's Miller values, bad = the OR of its items' status bits
HD uint8_t core_av_verdict(const fp12& F, uint32_t bad, bool nonempty) {
    if (!nonempty || bad) return 0;
    return fp12_is_one(final_exponentiation(F)) ? 1 : 0;
}

// ---- random-linear-combination batch verification (SURVEY.md section 8(f)-4, section 2 K6 "optional RLC batch mode")
// Instead of n independent checks e(PK_i, H_i) * e(-g1, S_i) == 1, one check per group of aggregates:
//     prod_i e([r_i] PK_i, H_i)  *  e(-g1, sum_i [r_i] S_i)  ==  1
// with 64-bit scalars r_i the signer cannot predict (they are derived from a verifier-chosen secret seed): one Miller loop
// and ONE final exponentiation per group instead of one of each per aggregate.  A group that fails is re-verified aggregate
// by aggregate, so every verdict is the one the per-aggregate rule gives (a false accept needs a 2^-63 coincidence).
HD uint64_t core_rlc_scalar(const uint8_t* seed32, uint32_t i, const uint8_t* msg32) {
    uint8_t buf[68], out[32];
#pragma unroll 1
    for (int k = 0; k < 32; k++) {
        buf[k] = seed32[k];
        buf[36 + k] = msg32[k];
    }
    buf[32] = (uint8_t)i;
    buf[33] = (uint8_t)(i >> 8);
    buf[34] = (uint8_t)(i >> 16);
    buf[35] = (uint8_t)(i >> 24);
    sha256_ctx c;
    sha256_init(c);
    sha256_update(c, buf, 68);
    sha256_final(c, out);
    uint64_t r = 0;
#pragma unroll 1
    for (int k = 7; k >= 0; k--) r = (r << 8) | out[k];
    return r | 1ull;                            // never zero
}
// [k]P for a per-thread 64-bit scalar: branch-free double-and-always-add
template <class F> HDN jac<F> pt_mul_var64(const jac<F>& p, uint64_t k) {
    jac<F> r = pt_inf<F>();
#pragma unroll 1
    for (int i = 63; i >= 0; i--) {
        r = pt_dbl(r);
        jac<F> s = pt_add(r, p);
        r = pt_select(((k >> i) & 1ull) != 0, s, r);
    }
    return r;
}
template <class F> HDN jac<F> pt_mul_var64_aff(const aff<F>& p, uint64_t k) {
    jac<F> r = pt_inf<F>();
#pragma unroll 1
    for (int i = 63; i >= 0; i--) {
        r = pt_dbl(r);
        jac<F> s = pt_add_mixed(r, p);
        r = pt_select(((k >> i) & 1ull) != 0, s, r);
    }
    return r;
}
// is aggregate a part of its group's batch equation?  (a bad key set or an undecodable / non-G2 signature is rejected outright)
HD bool rlc_in_batch(uint8_t pk_status, uint8_t sflag) { return pk_status == PK_OK && sflag != SIG_INVALID; }
// group verdict: F = f_sig * prod f_pk[i] over the batch members; no member -> nothing to prove
HD uint8_t core_rlc_group_verdict(const fp12& f_sig, const fp12* f_pk, const uint8_t* in_batch, uint32_t n) {
    fp12 F = f_sig;
    bool any = false;
#pragma unroll 1
    for (uint32_t i = 0; i < n; i++)
        if (in_batch[i]) {
            F = fp12_mul(F, f_pk[i]);
            any = true;
        }
    if (!any) return 1;
    return fp12_is_one(final_exponentiation(F)) ? 1 : 0;
}

// ---- SSZ: compute_signing_root(AttestationData, domain) (see k_signing_roots in kernels.cuh)
HD void sha256_pair(const uint8_t* left32, const uint8_t* right32, uint8_t* out32) {
    sha256_ctx c;
    sha256_init(c);
    sha256_update(c, left32, 32);
    sha256_update(c, right32, 32);
    sha256_final(c, out32);
}
// hash_tree_root(AttestationData) of its 128-byte serialisation
HD void attestation_data_root(const uint8_t* data128, uint8_t* root) {
    uint8_t chunk[8][32];
#pragma unroll 1
    for (int i = 0; i < 8; i++)
        for (int k = 0; k < 32; k++) chunk[i][k] = 0;
    uint8_t ep[32];
    for (int k = 0; k < 8; k++) {
        chunk[0][k] = data128[k];            // slot
        chunk[1][k] = data128[8 + k];        // index
    }
    for (int k = 0; k < 32; k++) chunk[2][k] = data128[16 + k];
    for (int k = 0; k < 32; k++) ep[k] = k < 8 ? data128[48 + k] : 0;
    sha256_pair(ep, data128 + 56, chunk[3]);     // htr(source)
    for (int k = 0; k < 32; k++) ep[k] = k < 8 ? data128[88 + k] : 0;
    sha256_pair(ep, data128 + 96, chunk[4]);     // htr(target)
    uint8_t l1[4][32], l2[2][32];
#pragma unroll 1
    for (int i = 0; i < 4; i++) sha256_pair(chunk[2 * i], chunk[2 * i + 1], l1[i]);
    sha256_pair(l1[0], l1[1], l2[0]);
    sha256_pair(l1[2], l1[3], l2[1]);
    sha256_pair(l2[0], l2[1], root);
}
HD void attestation_signing_root(const uint8_t* data128, const uint8_t* domain32, uint8_t* out32) {
    uint8_t root[32];
    attestation_data_root(data128, root);
    sha256_pair(root, domain32, out32);
}

}  // namespace b2
