"""The lazily reduced Fp forms of csrc/fp.cuh on the CPU (tests/hostsim/fp_lazy_sim.cpp): fp_mul_lazy / fp_sqr_lazy on inputs in
[0, 2p), compared bit for bit with the exact Montgomery quotient computed with Python integers, and the fixed-exponent chain
(fp_pow_prog, whose table and steps stay in [0, 2p)) on inputs at the ends of both ranges."""
import ctypes
import os
import random
import shutil
import subprocess
import tempfile

import numpy as np

import hs
from oracle.bls12_381 import P

R = 1 << 384
PINV = pow(P, -1, R)
rnd = random.Random(381)


def _build():
    """g++ build of tests/hostsim/fp_lazy_sim.cpp in a temporary directory: the tree is not written"""
    root = os.path.dirname(hs.HERE)
    d = tempfile.mkdtemp(prefix="fp_lazy_sim_")
    try:
        out = os.path.join(d, "libfp_lazy_sim.so")
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-x", "c++", "-I", os.path.join(root, "pos_evolution_b200", "csrc"),
                               os.path.join(hs.HERE, "hostsim", "fp_lazy_sim.cpp"), "-o", out])
        return ctypes.CDLL(out)
    finally:
        shutil.rmtree(d, ignore_errors=True)      # the loaded library stays mapped


lib = _build()


def arr(v):
    return np.array(hs.limbs(v), dtype=np.uint32)


def val(a):
    return sum(int(x) << (32 * i) for i, x in enumerate(a))


def redc(t):
    """the word-serial Montgomery quotient (t + M*p) / R with M = -t/p mod R: what both reductions compute, before any subtraction"""
    return (t + (-t * PINV % R) * P) >> 384


def mul(fn, a, b):
    out = np.zeros(12, dtype=np.uint32)
    fn(hs.ptr(arr(a)), hs.ptr(arr(b)), hs.ptr(out))
    return val(out)


def sqr(fn, a):
    out = np.zeros(12, dtype=np.uint32)
    fn(hs.ptr(arr(a)), hs.ptr(out))
    return val(out)


# raw limb values across [0, 2p): both ends of [0, p) and of [p, 2p), limb patterns, Montgomery images of small values
EDGE = [0, 1, 2, P - 2, P - 1, P, P + 1, P + 2, 2 * P - 2, 2 * P - 1, (P - 1) // 2, (P + 1) // 2, P + (P - 1) // 2, 1 << 380, 1 << 381,
        (1 << 381) - 1, 2 * P - 3, int("ffffffff" * 11, 16), P + int("ffffffff" * 11, 16),
        R % P, R % P + P, (1 << 352) - 1, P + (1 << 352)]
assert all(0 <= v < 2 * P for v in EDGE)


def r2p():
    return rnd.randrange(2 * P)


def rhigh():
    return P + rnd.randrange(P)


def test_lazy_sqr_exact_on_0_2p():
    for a in EDGE + [r2p() for _ in range(3000)] + [rhigh() for _ in range(2000)] + [2 * P - 1 - rnd.randrange(1 << 64) for _ in range(500)]:
        want = redc(a * a)
        assert want < 2 * P
        assert sqr(lib.hs_fp_sqr_lazy, a) == want, hex(a)
        assert sqr(lib.hs_fp_sqr, a) == (want - P if want >= P else want)


def test_lazy_mul_exact_on_0_2p():
    pairs = [(a, b) for a in EDGE for b in EDGE] + [(r2p(), r2p()) for _ in range(3000)] + [(rhigh(), rhigh()) for _ in range(2000)]
    pairs += [(2 * P - 1 - rnd.randrange(1 << 64), 2 * P - 1 - rnd.randrange(1 << 64)) for _ in range(500)]
    for a, b in pairs:
        want = redc(a * b)
        assert want < 2 * P
        assert mul(lib.hs_fp_mul_lazy, a, b) == want, (hex(a), hex(b))
        assert mul(lib.hs_fp_mul, a, b) == (want - P if want >= P else want)


def test_lazy_sqr_is_lazy_mul_of_a_by_a():
    """the dedicated squaring and the CIOS multiplication compute the same quotient, not just the same residue"""
    for a in EDGE + [r2p() for _ in range(1000)]:
        assert sqr(lib.hs_fp_sqr_lazy, a) == mul(lib.hs_fp_mul_lazy, a, a)


def test_chain_on_range_ends():
    """fp_pow_prog runs its table and steps on the lazy forms and reduces once: the result is the canonical Montgomery image of
    x^e, for x anywhere in [0, 2p) (as raw limbs: x stands for x/R mod p)"""
    exps = {0: (P - 3) // 4, 1: P - 2}
    xs = [0, 1, P - 1, P - 2, P, P + 1, 2 * P - 1, 2 * P - 2, R % P, (R % P) + P, P - (1 << 32)] + [r2p() for _ in range(6)] + [rhigh() for _ in range(6)]
    for which, e in exps.items():
        for x in xs:
            out = np.zeros(12, dtype=np.uint32)
            lib.hs_fp_pow_prog(hs.ptr(arr(x)), which, hs.ptr(out))
            assert val(out) == pow(x, e, P) * pow(R, 1 - e, P) % P, (which, hex(x))
