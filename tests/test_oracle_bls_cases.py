"""The adversarial BLS inputs of tests/bls_cases.py are what their names claim (so that no GPU test built on them can pass without
reaching the branch it targets), and the host-sim build of csrc/curve.cuh decodes every one of them as the oracle does."""
import ctypes

import numpy as np

import bls_cases as bc
import hs
from oracle import bls_sig as B
from oracle.bls12_381 import (P, HALF_P, E1, E2, G1, f2_neg, f2_sqrt, fp_sqrt, g1_compress, g1_decompress, g1_in_subgroup, g2_compress,
                              g2_decompress, g2_in_subgroup, pairing)

lib = hs.load()


def _g2_status(enc):
    return bc.decode_status(g2_decompress, enc)


def test_g2_encodings_are_what_they_claim():
    enc = dict(bc.g2_encodings())
    ok = {n for n, e in enc.items() if _g2_status(e) == 0}
    assert ok == {"valid", "sig_times_3", "torsion_t2", "sig_plus_t2", "not_in_g2"} | \
        {n for n, _ in bc.special_points_g2()} | {n + "_neg" for n, _ in bc.special_points_g2()}
    assert _g2_status(enc["infinity"]) == 1
    for n, e in enc.items():
        if n not in ok and n != "infinity":
            assert _g2_status(e) == 2, n
    # the rejected flag cases differ from an accepted encoding in the flags or the infinity payload only
    assert enc["compression_flag_clear"][1:] == enc["valid"][1:] and enc["compression_flag_clear"][0] & 0x80 == 0
    for n in ("c_i_byte47", "c_i_byte48", "c_i_byte95"):
        assert enc[n][0] == 0xC0 and sum(1 for b in enc[n][1:] if b) == 1
    # out-of-range x: one coordinate >= p, the other a valid signature's
    sx = E2.to_affine(g2_decompress(enc["valid"]))[0]
    for n, c1 in (("x1_eq_p", P), ("x1_eq_p_plus_1", P + 1), ("x1_all_ones", (1 << 381) - 1)):
        assert int.from_bytes(enc[n][:48], "big") & ((1 << 381) - 1) == c1 and int.from_bytes(enc[n][48:], "big") == sx[0]
    assert int.from_bytes(enc["x0_eq_p"][48:], "big") == P
    for bit in (381, 382, 383):
        assert int.from_bytes(enc["x0_top_bit_%d" % bit][48:], "big") >> bit & 1
    # the aliases: exactly the encoding of a valid signature with one coordinate raised by p, still below 2^381, so that only the
    # range check rejects them
    for n, lo, hi in (("x0_alias_plus_p", 48, 96), ("x1_alias_plus_p", 0, 48)):
        e = bytearray(enc[n])
        flags = e[0] & 0xE0
        v = int.from_bytes(e[lo:hi], "big") & ((1 << 381) - 1)
        assert P <= v < (1 << 381)
        e[lo:hi] = (v - P).to_bytes(48, "big")
        e[0] |= flags
        canon = bytes(e)
        assert _g2_status(canon) == 0 and g2_in_subgroup(g2_decompress(canon))
    # x = 0: 4 + 4i is not a square; the other off-curve x likewise
    assert f2_sqrt((4, 4)) is None
    for n, e in enc.items():
        if n.startswith("off_curve") or n.startswith("x_zero"):
            x = (int.from_bytes(e[48:], "big"), int.from_bytes(e[:48], "big") & ((1 << 381) - 1))
            assert x[0] < P and x[1] < P and f2_sqrt(bc.g2_rhs(x)) is None, n


def test_special_g2_points_take_the_branches_they_name():
    pts = dict(bc.special_points_g2())
    for name, (x, y) in pts.items():
        assert E2.on_curve_affine(x, y) and not g2_in_subgroup(E2.from_affine(x, y)), name
    # x^3 + 4 + 4i in Fp: a residue (root y = (y0, 0)) and a non-residue (root y = (0, y1)), both sign bits
    x, y = pts["rhs_fp_residue"]
    rhs = bc.g2_rhs(x)
    assert rhs[1] == 0 and fp_sqrt(rhs[0]) is not None and y[1] == 0 and y[0] != 0
    x, y = pts["rhs_fp_nonresidue"]
    rhs = bc.g2_rhs(x)
    assert rhs[1] == 0 and fp_sqrt(rhs[0]) is None and y[0] == 0 and y[1] != 0
    assert bc.rhs_c1_zero_x(19) == pts["rhs_fp_residue"][0] and bc.rhs_c1_zero_x(5) == pts["rhs_fp_nonresidue"][0]
    x, y = pts["rhs_c0_zero"]
    rhs = bc.g2_rhs(x)
    assert rhs[0] == 0 and rhs[1] != 0
    # lexicographic boundary: y.c1 = (p-1)/2 exactly (not the larger root); y = (c0, 0) decided by c0 alone
    x, y = pts["y_c1_half"]
    assert y == (4, HALF_P)
    x, y = pts["y_c0_near_half"]
    assert y[1] == 0 and abs(y[0] - HALF_P) < 64
    # the sign bit of each encoding picks the y of its name
    enc = dict(bc.g2_encodings())
    for name, (x, y) in pts.items():
        assert E2.to_affine(g2_decompress(enc[name])) == (x, y)
        assert E2.to_affine(g2_decompress(enc[name + "_neg"])) == (x, f2_neg(y))
    assert enc["y_c1_half"][0] & 0x20 == 0 and enc["y_c1_half_neg"][0] & 0x20


def test_g1_encodings_are_what_they_claim():
    enc = dict(bc.g1_encodings())
    st = {n: bc.decode_status(g1_decompress, e) for n, e in enc.items()}
    assert {n for n, s in st.items() if s == 0} == {"valid", "order3_y2", "order3_y_minus_2", "not_in_g1", "not_in_g1_neg", "torsion_t1", "pk_plus_t1"}
    assert st["infinity"] == 1
    assert [n for n in enc if B.KeyValidate(enc[n])] == ["valid"]
    assert E1.to_affine(g1_decompress(enc["order3_y2"])) == (0, 2) and E1.to_affine(g1_decompress(enc["order3_y_minus_2"])) == (0, P - 2)
    assert E1.is_inf(E1.mul(g1_decompress(enc["order3_y2"]), 3))
    t1 = bc.t1()
    assert not E1.is_inf(t1) and not g1_in_subgroup(t1)
    e = bytearray(enc["x_alias_plus_p"])
    v = int.from_bytes(e, "big") & ((1 << 381) - 1)
    assert P <= v < (1 << 381)
    canon = bytearray((v - P).to_bytes(48, "big"))
    canon[0] |= e[0] & 0xE0
    assert B.KeyValidate(bytes(canon))
    (n0, (x0, y0)), (n1, (x1, y1)) = bc.boundary_points_g1()
    assert x0 == x1 and y0 == HALF_P - 4 and y1 == HALF_P + 5 and E1.on_curve_affine(x0, y0)
    for d in range(4):                                  # and no point lies closer to (p-1)/2 from below
        assert bc.fp_cube_root(((HALF_P - d) ** 2 - 4) % P) is None


def test_torsion_constructions():
    t2 = bc.t2()
    s1, s2 = bc.sig_point(bc.sk(1)), bc.sig_point(bc.sk(2))
    assert not E2.is_inf(t2) and not g2_in_subgroup(t2)
    a, b = E2.add(s1, t2), E2.add(s2, E2.neg(t2))
    assert not g2_in_subgroup(a) and not g2_in_subgroup(b) and g2_in_subgroup(E2.add(a, b))
    assert not g2_in_subgroup(E2.add(a, s2))
    # S + T2 is rejected by the pairing on its own as well (so dropping a subgroup test cannot be seen through a verdict)
    assert pairing(G1, a) != pairing(G1, s1)
    assert not B.FastAggregateVerify([B.SkToPk(bc.sk(1))], bc.MSG, g2_compress(a))
    agg = B.Aggregate([g2_compress(a), g2_compress(s2)])
    assert not g2_in_subgroup(g2_decompress(agg))
    pk12 = [B.SkToPk(bc.sk(1)), B.SkToPk(bc.sk(2))]
    assert not B.FastAggregateVerify(pk12, bc.MSG, agg)
    assert B.FastAggregateVerify(pk12, bc.MSG, B.Aggregate([g2_compress(a), g2_compress(b)]))


def test_sharp_cases_pass_the_pairing_alone():
    rows, index = bc.registry()
    for c in bc.sharp_registry_cases():
        assert bc.pairing_alone(c["blind_pk"], g2_decompress(c["sig"]), c["msg"]), c["name"]
        sel = [rows[index[m]] for m, b in zip(c["members"], c["bits"]) if b]
        assert bc.fav(sel, c["msg"], c["sig"]) is False, c["name"]
    for c in bc.sharp_explicit_cases():
        assert bc.pairing_alone(c["blind_pk"], g2_decompress(c["sig"]), c["msg"]), c["name"]
        assert not any(B.KeyValidate(p) for p in c["pks"][1:]) and bc.fav(c["pks"], c["msg"], c["sig"]) is False, c["name"]
    shifted = bc.sharp_explicit_cases()[0]
    assert not B.KeyValidate(shifted["pks"][0]) and E1.eq(shifted["blind_pk"], bc.g1_points_sum([g1_decompress(p) for p in shifted["pks"]]))
    want = {"sig_then_undecodable_one_bit": (1, False), "torsion_cancels_in_sum": (0, True)}
    for c in bc.sharp_aggregation_cases():
        pk, sig = c["blind"]
        assert bc.pairing_alone(pk, sig, bc.MSG), c["name"]
        st, agg = bc.aggregate(c["sigs"])
        sel = [rows[index[m]] for m, b in zip(c["members"], c["bits"]) if b]
        assert (st, st == 0 and bc.fav(sel, bc.MSG, agg)) == want[c["name"]], c["name"]


def test_registry_rows():
    rows, index = bc.registry()
    assert len(set(rows[:2 * bc.N_HONEST])) == 2 * bc.N_HONEST
    valid = [B.KeyValidate(r) for r in rows]
    assert valid[:2 * bc.N_HONEST] == [True] * (2 * bc.N_HONEST)
    assert sum(valid) == 2 * bc.N_HONEST + 1                        # + enc:valid
    s = E1.add(g1_decompress(rows[index["pk1+t1"]]), g1_decompress(rows[index["pk2-t1"]]))
    assert E1.eq(s, E1.add(bc.pk_point(1), bc.pk_point(2)))


def test_patterns_reach_the_exceptional_additions():
    """the group-law segments sum to what the oracle's Aggregate says, and each contains equal or opposite points"""
    for name, sigs in bc.g2_patterns():
        st, agg = bc.aggregate(sigs)
        if name == "empty":
            assert st == 2
        elif name == "sig_then_undecodable":
            assert st == 1
        else:
            assert st == 0, name
        if name.startswith("alternating_1026") or name.startswith("halves") or name in ("alternating_64",):
            assert agg == bc.INF2, name
    rows, index = bc.registry()
    for name, members, bits in bc.g1_patterns():
        st, out = bc.g1_pattern_sum(rows, index, members, bits)
        assert st & 3 == 0, name


# ------------------------------------------------------------------------------------------ host-sim decoders vs the oracle
def _hs_g2(enc):
    out = np.zeros(48, dtype=np.uint32)
    s = lib.hs_g2_decompress(hs.buf(enc), hs.ptr(out))
    return s, (hs.fp2_v(out[:24]), hs.fp2_v(out[24:]))


def _hs_g1(enc):
    out = np.zeros(24, dtype=np.uint32)
    s = lib.hs_g1_decompress(hs.buf(enc), hs.ptr(out))
    return s, (hs.fp_v(out[:12]), hs.fp_v(out[12:]))


def test_hostsim_g2_decompress_every_encoding():
    for name, enc in bc.g2_encodings():
        s, aff = _hs_g2(enc)
        want = _g2_status(enc)
        assert s == want, name
        if want == 0:
            assert aff == E2.to_affine(g2_decompress(enc)), name


def test_hostsim_g1_decompress_every_encoding():
    for name, enc in bc.g1_encodings() + bc.g1_boundary_encodings():
        s, aff = _hs_g1(enc)
        want = bc.decode_status(g1_decompress, enc)
        assert s == want, name
        if want == 0:
            assert aff == E1.to_affine(g1_decompress(enc)), name
    # and the sign bit the host-sim compressor gives the near-boundary pair (outside G1: not visible through the C ABI)
    for name, enc in bc.g1_boundary_encodings():
        o = ctypes.create_string_buffer(48)
        assert lib.hs_g1_add(hs.buf(enc), hs.buf(bc.INF1), o, 0) == 0 and o.raw == enc, name


def test_hostsim_exceptional_additions_and_compress():
    """Y - S + S == Y (compress of the special points), S + S (doubling branch) and S + (-S) (cancellation), mixed and Jacobian"""
    s = bc.sign(bc.sk(3))
    ns = g2_compress(E2.neg(bc.sig_point(bc.sk(3))))
    for mixed in (0, 1):
        o = ctypes.create_string_buffer(96)
        assert lib.hs_g2_add(hs.buf(s), hs.buf(s), o, mixed) == 0 and o.raw == g2_compress(E2.dbl(bc.sig_point(bc.sk(3))))
        assert lib.hs_g2_add(hs.buf(s), hs.buf(ns), o, mixed) == 0 and o.raw == bc.INF2
        for name, segment in bc.g2_patterns():
            if name.startswith("y_minus_s_plus_s:"):
                assert lib.hs_g2_add(hs.buf(segment[0]), hs.buf(segment[1]), o, mixed) == 0
                assert o.raw == B.Aggregate(segment), name
        pk = g1_compress(bc.pk_point(3))
        npk = g1_compress(E1.neg(bc.pk_point(3)))
        o1 = ctypes.create_string_buffer(48)
        assert lib.hs_g1_add(hs.buf(pk), hs.buf(pk), o1, mixed) == 0 and o1.raw == g1_compress(E1.dbl(bc.pk_point(3)))
        assert lib.hs_g1_add(hs.buf(pk), hs.buf(npk), o1, mixed) == 0 and o1.raw == bc.INF1
