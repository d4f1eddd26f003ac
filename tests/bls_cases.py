"""Adversarial BLS inputs for the GPU kernels, built on the CPU with the oracle (test-only).

Every expected value comes from the oracle (`B.Aggregate`, `B.FastAggregateVerify`, `B.KeyValidate`); nothing here is written
by hand.  tests/test_oracle_bls_cases.py proves that each construction is what its name claims (on the curve or not, which
square-root branch it takes, which y coordinate is zero, subgroup membership, and that the pairing alone accepts every "sharp"
case), so that no GPU test in tests/test_gpu_bls_adversarial.py can pass without exercising the branch it targets.

Contents:
  * G2 (96-byte) and G1 (48-byte) encodings: flag combinations, out-of-range and non-canonical x, x off the curve, points whose
    curve right-hand side lies in Fp (both square-root branches), a zero real part of the right-hand side, and y exactly at
    the lexicographic boundary (p - 1)/2;
  * torsion points T2 (E2, order divides the G2 cofactor) and T1 (E1, outside G1);
  * a small registry: honest keys, their negatives, every G1 encoding, and torsion-shifted keys;
  * group-law patterns that force the doubling and cancellation branches of the point additions however lanes are assigned;
  * "sharp" cases, on which the pairing equation alone accepts, so that only the status bit or rule they target rejects them.
"""
import contextlib
import functools
import hashlib

from oracle import bls_sig as B
from oracle.bls12_381 import (P, R, E1, E2, G1, HALF_P, DeserializationError, f2_add, f2_mul, f2_muls, f2_neg, f2_pow, f2_sqr, f2_sub,
                              fp_sqrt, g1_compress, g1_decompress, g2_compress, g2_decompress, pairing_product_is_one)
from oracle.hash_to_curve import hash_to_g2, map_to_curve_g2

INF1 = bytes([0xC0]) + bytes(47)
INF2 = bytes([0xC0]) + bytes(95)
MSG = hashlib.sha256(b"bls-cases/message").digest()
MSG2 = hashlib.sha256(b"bls-cases/other-message").digest()
# the k of "the same point k times": both sides of the warp width, of a 4-warp block and of the gather chunk
REPEATS = (2, 31, 32, 33, 64, 65, 128, 129, 513, 1025)
C, I, S = 0x80, 0x40, 0x20          # ZCash flag bits of byte 0: compressed, infinity, sign (y lexicographically largest)


def sk(i: int) -> int:
    return int.from_bytes(hashlib.sha256(b"bls-cases/sk%d" % i).digest(), "big") % R or 1


@functools.cache
def h_msg(msg: bytes = MSG):
    return hash_to_g2(msg)


@functools.cache
def sig_point(k: int, msg: bytes = MSG):
    """[k] H(msg): the signature of secret key k (k taken mod r)"""
    return E2.mul(h_msg(msg), k % R)


def sign(k: int, msg: bytes = MSG) -> bytes:
    return g2_compress(sig_point(k, msg))


@functools.cache
def pk_point(i: int):
    return E1.mul(G1, sk(i))


def g2_bytes(x0: int, x1: int, flags: int) -> bytes:
    """x.c1 || x.c0, big endian, flags OR-ed into byte 0 (no range or curve check)"""
    b = bytearray(x1.to_bytes(48, "big") + x0.to_bytes(48, "big"))
    b[0] |= flags
    return bytes(b)


def g1_bytes(x: int, flags: int) -> bytes:
    b = bytearray(x.to_bytes(48, "big"))
    b[0] |= flags
    return bytes(b)


def decode_status(dec, enc: bytes) -> int:
    """0 = point, 1 = infinity, 2 = undecodable (the DecodeStatus of csrc/curve.cuh), by the oracle"""
    try:
        p = dec(enc)
    except DeserializationError:
        return 2
    return 1 if (E2 if len(enc) == 96 else E1).is_inf(p) else 0


# ------------------------------------------------------------------------------------------ cube roots (p = 1 mod 9, p != -1 mod 3)
def _zeta9():
    """a primitive 9th root of unity in Fp (9 divides p - 1 exactly)"""
    g = 2
    while True:
        z = pow(g, (P - 1) // 9, P)
        if pow(z, 3, P) != 1:
            return z
        g += 1


def fp_cube_root(u: int):
    m = (P - 1) // 9
    c = pow(u, pow(3, -1, m), P)
    z = _zeta9()
    for i in range(9):
        cand = c * pow(z, i, P) % P
        if pow(cand, 3, P) == u % P:
            return cand
    return None


def f2_cube_root(u):
    """the 3-part of p^2 - 1 is 9 (9 || p - 1, 3 does not divide p + 1): u^(1/3 mod (p^2-1)/9) times a 9th root of unity"""
    m = (P * P - 1) // 9
    c = f2_pow(u, pow(3, -1, m))
    z = _zeta9()
    for i in range(9):
        cand = f2_muls(c, pow(z, i, P))
        if f2_pow(cand, 3) == (u[0] % P, u[1] % P):
            return cand
    return None


def g2_rhs(x):
    return f2_add(f2_mul(f2_sqr(x), x), (4, 4))


# ------------------------------------------------------------------------------------------ special curve points
@functools.cache
def rhs_c1_zero_x(b: int):
    """x = (a, b) with a = sqrt((b^2 - 4/b)/3): then x^3 + 4 + 4i lies in Fp"""
    a = fp_sqrt((b * b - 4 * pow(b, -1, P)) * pow(3, -1, P) % P)
    assert a is not None, b
    return (a, b)


@functools.cache
def rhs_c0_zero_x():
    """x = (a, b) with a^3 - 3ab^2 + 4 = 0 (real part of x^3 + 4 + 4i zero) and x^3 + 4 + 4i a square: the smallest such a"""
    a = 1
    while True:
        b = fp_sqrt((a * a * a + 4) * pow(3 * a, -1, P) % P)
        if b is not None:
            try:
                g2_decompress(g2_bytes(a, b, C))
                return (a, b)
            except DeserializationError:
                pass
        a += 1


@functools.cache
def boundary_points_g2():
    """affine points of E2 whose y sits exactly at the lexicographic boundary:
    y = (4, (p-1)/2) (decided by c1), and y = (c0, 0) with c0 the value nearest (p-1)/2 for which y^2 - 4 - 4i is a cube
    (decided by c0 through the c1 == 0 fallback)"""
    out = []
    y = (4, HALF_P)
    x = f2_cube_root(f2_sub(f2_sqr(y), (4, 4)))
    assert x is not None
    out.append(("y_c1_half", (x, y)))
    for d in range(0, 64):
        for c0 in ((HALF_P - d, HALF_P + d) if d else (HALF_P,)):
            y = (c0, 0)
            x = f2_cube_root(f2_sub(f2_sqr(y), (4, 4)))
            if x is not None:
                out.append(("y_c0_near_half", (x, y)))
                return out
    raise AssertionError("no cube near (p-1)/2")


@functools.cache
def special_points_g2():
    """name -> affine point of E2 (not in G2): the c1 == 0 right-hand sides (square and non-square in Fp), a zero real part, and
    the boundary points"""
    pts = []
    for name, b in (("rhs_fp_residue", 19), ("rhs_fp_nonresidue", 5)):
        x = rhs_c1_zero_x(b)
        pts.append((name, E2.to_affine(g2_decompress(g2_bytes(x[0], x[1], C)))))
    x = rhs_c0_zero_x()
    pts.append(("rhs_c0_zero", E2.to_affine(g2_decompress(g2_bytes(x[0], x[1], C)))))
    pts += boundary_points_g2()
    return pts


@functools.cache
def g1_outside_point():
    """a point of E1 outside the r-torsion (the smallest x that gives one)"""
    x = 1
    while True:
        try:
            p = g1_decompress(g1_bytes(x, C))
            if not E1.is_inf(E1.mul(p, R)):
                return p
        except DeserializationError:
            pass
        x += 1


@functools.cache
def boundary_points_g1():
    """no point of E1 has y = (p-1)/2; the nearest below it, and its negative (just above)"""
    for d in range(0, 64):
        y = HALF_P - d
        x = fp_cube_root((y * y - 4) % P)
        if x is not None:
            return [("y_half_minus_%d" % d, (x, y)), ("y_half_plus_%d" % (d + 1), (x, P - y))]
    raise AssertionError("no point near (p-1)/2")


@functools.cache
def t2():
    """[r] map_to_curve_g2((13, 14)): a non-zero point whose order divides the G2 cofactor"""
    return E2.mul(map_to_curve_g2((13, 14)), R)


@functools.cache
def t1():
    """[r] Q for Q on E1 outside G1: a non-zero point whose order divides the G1 cofactor"""
    return E1.mul(g1_outside_point(), R)


def _aff_g2(p):
    return E2.from_affine(*p)


# ------------------------------------------------------------------------------------------ encoding tables
@functools.cache
def g2_encodings():
    """[(name, 96 bytes)]: every case's oracle decode status is decode_status(g2_decompress, bytes)"""
    s = sign(sk(0))
    sx = E2.to_affine(g2_decompress(s))[0]
    room = (1 << 381) - P
    alias0 = next(i for i in range(1, 200) if E2.to_affine(sig_point(sk(i)))[0][0] < room)
    alias1 = next(i for i in range(1, 200) if E2.to_affine(sig_point(sk(i)))[0][1] < room)
    a0, a1 = E2.to_affine(sig_point(sk(alias0)))[0], E2.to_affine(sig_point(sk(alias1)))[0]
    out = [
        ("valid", s),
        ("sig_times_3", g2_compress(E2.mul(sig_point(sk(1)), 3))),
        ("infinity", INF2),
        ("zero_bytes", bytes(96)),
        ("compression_flag_clear", bytes([s[0] & 0x7F]) + s[1:]),
        ("c_i_s", bytes([C | I | S]) + bytes(95)),
        ("c_i_byte47", bytes([C | I]) + bytes(46) + b"\x01" + bytes(48)),
        ("c_i_byte48", bytes([C | I]) + bytes(47) + b"\x01" + bytes(47)),
        ("c_i_byte95", bytes([C | I]) + bytes(94) + b"\x01"),
        ("i_without_c", bytes([I]) + bytes(95)),
        ("x1_eq_p", g2_bytes(sx[0], P, C)),
        ("x1_eq_p_plus_1", g2_bytes(sx[0], P + 1, C)),
        ("x1_all_ones", g2_bytes(sx[0], (1 << 381) - 1, C)),
        ("x0_eq_p", g2_bytes(P, sx[1], C)),
        ("x0_top_bit_381", g2_bytes(sx[0] | (1 << 381), sx[1], C)),
        ("x0_top_bit_382", g2_bytes(sx[0] | (1 << 382), sx[1], C)),
        ("x0_top_bit_383", g2_bytes(sx[0] | (1 << 383), sx[1], C)),
        ("x0_alias_plus_p", g2_bytes(a0[0] + P, a0[1], g2_compress(sig_point(sk(alias0)))[0] & 0xE0)),
        ("x1_alias_plus_p", g2_bytes(a1[0], a1[1] + P, g2_compress(sig_point(sk(alias1)))[0] & 0xE0)),
        ("x_zero", g2_bytes(0, 0, C)),
        ("x_zero_sign", g2_bytes(0, 0, C | S)),
    ]
    # further x off the curve: the first few small x = (k, 0) and (0, k) whose right-hand side is not a square
    for name, mk in (("x_real", lambda k: (k, 0)), ("x_imag", lambda k: (0, k))):
        k, found = 1, 0
        while found < 2:
            x = mk(k)
            if decode_status(g2_decompress, g2_bytes(x[0], x[1], C)) == 2:
                out.append(("off_curve_%s_%d" % (name, k), g2_bytes(x[0], x[1], C)))
                found += 1
            k += 1
    for name, (x, y) in special_points_g2():
        out.append((name, g2_compress(_aff_g2((x, y)))))
        out.append((name + "_neg", g2_compress(_aff_g2((x, f2_neg(y))))))
    out.append(("torsion_t2", g2_compress(t2())))
    out.append(("sig_plus_t2", g2_compress(E2.add(sig_point(sk(0)), t2()))))
    out.append(("not_in_g2", g2_compress(map_to_curve_g2((3, 4)))))
    return out


@functools.cache
def g1_encodings():
    """[(name, 48 bytes)]"""
    pk = B.SkToPk(sk(0))
    x = g1_decompress(pk)[0]
    room = (1 << 381) - P
    alias = next(i for i in range(1, 200) if E1.to_affine(pk_point(i))[0] < room)
    ax, ay = E1.to_affine(pk_point(alias))
    q = E1.to_affine(g1_outside_point())
    out = [
        ("valid", pk),
        ("infinity", INF1),
        ("zero_bytes", bytes(48)),
        ("compression_flag_clear", bytes([pk[0] & 0x7F]) + pk[1:]),
        ("c_i_s", bytes([C | I | S]) + bytes(47)),
        ("c_i_byte47", bytes([C | I]) + bytes(46) + b"\x01"),
        ("c_i_byte1", bytes([C | I, 1]) + bytes(46)),
        ("i_without_c", bytes([I]) + bytes(47)),
        ("x_eq_p", g1_bytes(P, C)),
        ("x_eq_p_plus_1", g1_bytes(P + 1, C)),
        ("x_all_ones", g1_bytes((1 << 381) - 1, C)),
        ("x_alias_plus_p", g1_bytes(ax + P, C | (S if ay > HALF_P else 0))),
        ("order3_y2", g1_bytes(0, C)),
        ("order3_y_minus_2", g1_bytes(0, C | S)),
        ("not_in_g1", g1_compress(E1.from_affine(*q))),
        ("not_in_g1_neg", g1_compress(E1.neg(E1.from_affine(*q)))),
        ("torsion_t1", g1_compress(t1())),
        ("pk_plus_t1", g1_compress(E1.add(pk_point(1), t1()))),
    ]
    k = 1
    while True:
        if decode_status(g1_decompress, g1_bytes(x + k, C)) == 2:
            out.append(("off_curve", g1_bytes(x + k, C)))
            break
        k += 1
    return out


def g1_boundary_encodings():
    """the near-boundary pair: outside G1, so only the host-sim decoder can show their sign bit"""
    return [(name, g1_compress(E1.from_affine(x, y))) for name, (x, y) in boundary_points_g1()]


# ------------------------------------------------------------------------------------------ registry
N_HONEST = 24


@functools.cache
def registry():
    """(rows: [48 bytes], index: name -> row).  Rows 0..N_HONEST-1 honest keys, then their negatives ("neg<i>"), every G1
    encoding ("enc:<name>") and the torsion-shifted keys pk1 + T1, pk2 - T1 (each outside G1; their sum is pk1 + pk2)."""
    rows, index = [], {}
    for i in range(N_HONEST):
        index["pk%d" % i] = len(rows)
        rows.append(g1_compress(pk_point(i)))
    for i in range(N_HONEST):
        index["neg%d" % i] = len(rows)
        rows.append(g1_compress(E1.neg(pk_point(i))))
    for name, enc in g1_encodings():
        index["enc:" + name] = len(rows)
        rows.append(enc)
    index["pk1+t1"] = len(rows)
    rows.append(g1_compress(E1.add(pk_point(1), t1())))
    index["pk2-t1"] = len(rows)
    rows.append(g1_compress(E1.add(pk_point(2), E1.neg(t1()))))
    return rows, index


# ------------------------------------------------------------------------------------------ oracle, memoised
_KV = {}


@contextlib.contextmanager
def cached_key_validate():
    """B.FastAggregateVerify with B.KeyValidate memoised by key bytes (a committee that repeats one key 1025 times would otherwise
    repeat its subgroup check 1025 times); the verdicts are B.FastAggregateVerify's own"""
    orig = B.KeyValidate

    def kv(pk):
        pk = bytes(pk)
        if pk not in _KV:
            _KV[pk] = orig(pk)
        return _KV[pk]

    B.KeyValidate = kv
    try:
        yield
    finally:
        B.KeyValidate = orig


_FAV = {}


def fav(pks, msg: bytes, sig: bytes) -> bool:
    key = (tuple(bytes(p) for p in pks), bytes(msg), bytes(sig))
    if key not in _FAV:
        with cached_key_validate():
            _FAV[key] = B.FastAggregateVerify(list(key[0]), key[1], key[2])
    return _FAV[key]


def aggregate(sigs):
    """(status, bytes) as b2_aggregate reports them: B.Aggregate's result, or status 2 (empty) / 1 (undecodable) and zero bytes"""
    if not sigs:
        return 2, bytes(96)
    try:
        return 0, B.Aggregate(list(sigs))
    except DeserializationError:
        return 1, bytes(96)


# ------------------------------------------------------------------------------------------ group-law patterns
def g2_patterns():
    """[(name, [96-byte signatures])]: segments that force equal and opposite partial sums in every warp and block tree"""
    s = sign(sk(3))
    ns = g2_compress(E2.neg(sig_point(sk(3))))
    out = [("same_x%d" % k, [s] * k) for k in REPEATS]
    out += [("alternating_64", [s, ns] * 32), ("alternating_65", [s, ns] * 32 + [s]), ("alternating_1026", [s, ns] * 513),
            ("halves_64", [s] * 32 + [ns] * 32), ("halves_130", [s] * 65 + [ns] * 65), ("halves_1026", [s] * 513 + [ns] * 513),
            ("p_negp_p", [s, ns, s])]
    for name, (x, y) in special_points_g2():
        for yy, tag in ((y, ""), (f2_neg(y), "_neg")):
            yp = _aff_g2((x, yy))
            out.append(("y_minus_s_plus_s:" + name + tag, [g2_compress(E2.add(yp, E2.neg(sig_point(sk(3))))), s]))
    s1, s2 = sig_point(sk(1)), sig_point(sk(2))
    out.append(("torsion_s1t_s2", [g2_compress(E2.add(s1, t2())), g2_compress(s2)]))
    out.append(("torsion_s1t_s2mt", [g2_compress(E2.add(s1, t2())), g2_compress(E2.add(s2, E2.neg(t2())))]))
    out.append(("sig_then_undecodable", [g2_compress(s1), bytes(96)]))
    out.append(("empty", []))
    return out


def g1_patterns():
    """[(name, [registry names], [bits])]: committees over registry() with repeated members and rows holding -pk"""
    v, n = "pk5", "neg5"
    out = [("same_x%d" % k, [v] * k, [1] * k) for k in REPEATS]
    out += [("alternating_64", [v, n] * 32, [1] * 64), ("alternating_65", [v, n] * 32 + [v], [1] * 65),
            ("alternating_1026", [v, n] * 513, [1] * 1026), ("halves_64", [v] * 32 + [n] * 32, [1] * 64),
            ("halves_130", [v] * 65 + [n] * 65, [1] * 130), ("halves_1026", [v] * 513 + [n] * 513, [1] * 1026),
            ("p_negp_p", [v, n, v], [1] * 3),
            ("pair_sum_then_double", ["pk6", "pk7", "pk6", "pk7"] * 16, [1] * 64),
            ("every_other_bit", [v, n] * 40, [1, 0] * 40)]
    return out


def g1_pattern_sum(rows, index, names, bits):
    """(status, bytes) b2_g1_aggregate reports: bit 1 a selected invalid key (left out of the sum), 2 nothing selected, 4 sum = infinity"""
    acc, bad, cnt = E1.INF, False, 0
    for nm, b in zip(names, bits):
        if not b:
            continue
        cnt += 1
        pk = rows[index[nm]]
        with cached_key_validate():
            ok = B.KeyValidate(pk)
        if not ok:
            bad = True
            continue
        acc = E1.add(acc, g1_decompress(pk))
    return (1 if bad else 0) | (2 if cnt == 0 else 0) | (4 if E1.is_inf(acc) else 0), g1_compress(acc)


def g1_points_sum(pts):
    acc = E1.INF
    for p in pts:
        acc = E1.add(acc, p)
    return acc


# ------------------------------------------------------------------------------------------ sharp cases
# Each case: name, members (registry names), bits, msg, sig (96 bytes), blind_pk (the G1 point the pairing sees when the rule the
# case targets is missing: the sum the key aggregation forms, or None where the kernels substitute 1 for the key side), target.
# On every case pairing_product_is_one([(blind_pk, H(msg)), (-g1, sig)]) holds (tests/test_oracle_bls_cases.py), while the oracle
# verdict is False (or, for the last one, True): only the status bit or rule named in `target` decides.
def sharp_registry_cases():
    rows, index = registry()
    out = []
    for bad in ("enc:zero_bytes", "enc:infinity", "enc:not_in_g1"):
        out.append(dict(name="valid_plus_" + bad[4:], members=["pk8", bad], bits=[1, 1], msg=MSG, sig=sign(sk(8)),
                        blind_pk=pk_point(8), target="K2 marks the invalid key in status only"))
    out.append(dict(name="pk_negpk_sig_inf", members=["pk9", "neg9"], bits=[1, 1], msg=MSG, sig=INF2, blind_pk=None,
                    target="aggregate pubkey infinity: verdict status test"))
    out.append(dict(name="no_bits_sig_inf", members=["pk10", "pk11"], bits=[0, 0], msg=MSG, sig=INF2, blind_pk=None,
                    target="empty selection: verdict status test"))
    out.append(dict(name="valid_plus_invalid_sig_inf", members=["pk12", "enc:zero_bytes"], bits=[1, 1], msg=MSG, sig=INF2,
                    blind_pk=None, target="invalid key: verdict status test"))
    return out


def sharp_explicit_cases():
    """explicit-key path (b2_fast_aggregate_verify_pks): [48-byte keys]"""
    t = t1()
    p1, p2 = pk_point(13), pk_point(14)
    return [
        dict(name="torsion_shifted_keys", pks=[g1_compress(E1.add(p1, t)), g1_compress(E1.add(p2, E1.neg(t)))], msg=MSG,
             sig=sign(sk(13) + sk(14)), blind_pk=E1.add(p1, p2), target="every key is validated on its own"),
        dict(name="valid_plus_undecodable", pks=[g1_compress(p1), bytes(48)], msg=MSG, sig=sign(sk(13)), blind_pk=p1,
             target="k_g1_segment_sum marks the invalid key in status only"),
    ]


def sharp_aggregation_cases():
    """epoch path: (name, members, bits, individual signatures, blind (pk, sig point) or None, target)"""
    s15 = sig_point(sk(15))
    s16, s17 = sig_point(sk(16)), sig_point(sk(17))
    return [
        dict(name="sig_then_undecodable_one_bit", members=["pk15", "pk18"], bits=[1, 0], sigs=[g2_compress(s15), bytes(96)],
             blind=(pk_point(15), s15), target="k_g2_segment_sum marks DEC_BAD in seg_status only"),
        dict(name="torsion_cancels_in_sum", members=["pk16", "pk17"], bits=[1, 1],
             sigs=[g2_compress(E2.add(s16, t2())), g2_compress(E2.add(s17, E2.neg(t2())))], blind=(E1.add(pk_point(16), pk_point(17)), E2.add(s16, s17)),
             target="the subgroup test applies to the aggregate, not to each contribution"),
    ]


def pairing_alone(pk, sig_pt, msg):
    """e(pk, H(msg)) * e(-g1, sig) == 1, an infinite argument giving 1"""
    return pairing_product_is_one([(pk if pk is not None else E1.INF, h_msg(msg)), (E1.neg(G1), sig_pt)])
