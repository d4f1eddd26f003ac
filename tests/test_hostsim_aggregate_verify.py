"""bls.AggregateVerify on the CPU: the per-item bodies of csrc/aggverify.cuh (item -> set mapping, pair / signature Miller arguments,
per-set product and verdict in csrc/cores.cuh), looped on the host by tests/hostsim/aggverify_sim.cpp, against
oracle.bls_sig.AggregateVerify.  Small sets (1-4 pairs) keep this to seconds."""
import ctypes
import hashlib
import os
import shutil
import subprocess
import tempfile

import numpy as np

import bls_cases as bc
import hs
from oracle import bls_sig as B
from oracle.bls12_381 import E2, g2_compress


def _build():
    """g++ build of tests/hostsim/aggverify_sim.cpp (the csrc headers for the CPU) in a temporary directory: the tree is not written"""
    root = os.path.dirname(hs.HERE)
    d = tempfile.mkdtemp(prefix="aggverify_sim_")
    try:
        out = os.path.join(d, "libaggverify_sim.so")
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-x", "c++", "-I", os.path.join(root, "pos_evolution_b200", "csrc"),
                               os.path.join(hs.HERE, "hostsim", "aggverify_sim.cpp"), "-o", out])
        return ctypes.CDLL(out)
    finally:
        shutil.rmtree(d, ignore_errors=True)      # the loaded library stays mapped


lib = _build()
M =[hashlib.sha256(b"hostsim-av/%d" % i).digest() for i in range(4)]


def _pk(i):
    return B.SkToPk(bc.sk(i))


def _agg_sig(pairs):
    """the honest aggregate signature of [(key number, message)]"""
    return B.Aggregate([bc.sign(bc.sk(k), m) for k, m in pairs])


def _run(sets):
    """sets: [(pks, msgs, sig)] -> the host-sim verdicts"""
    pks = [p for s in sets for p in s[0]]
    msgs = [m for s in sets for m in s[1]]
    off = np.cumsum([0] + [len(s[0]) for s in sets]).astype(np.uint32)
    ok = np.full(len(sets), 9, dtype=np.uint8)
    lib.hs_core_aggregate_verify(hs.buf(b"".join(pks) or bytes(1)), hs.buf(b"".join(msgs) or bytes(1)), hs.ptr(off), hs.buf(b"".join(s[2] for s in sets)),
                                 len(sets), hs.ptr(ok))
    return ok.tolist()


def test_aggregate_verify_core_matches_oracle():
    valid = [(0, M[0]), (1, M[1]), (2, M[0])]                       # distinct and repeated messages
    swapped_sig = _agg_sig([(3, M[1]), (4, M[2])])
    sets = [
        ("valid_3", [_pk(k) for k, _ in valid], [m for _, m in valid], _agg_sig(valid)),
        ("empty", [], [], _agg_sig([(5, M[0])])),
        ("valid_1", [_pk(5)], [M[3]], bc.sign(bc.sk(5), M[3])),
        ("message_swapped", [_pk(3), _pk(4)], [M[2], M[1]], swapped_sig),
        ("key_off_curve", [_pk(6), dict(bc.g1_encodings())["off_curve"]], [M[0], M[1]], bc.sign(bc.sk(6), M[0])),
        ("torsion_sig", [_pk(0)], [bc.MSG], g2_compress(E2.add(bc.sig_point(bc.sk(0)), bc.t2()))),
        ("same_key_twice", [_pk(7), _pk(7), _pk(8), _pk(9)], [M[0], M[1], M[2], M[2]],
         _agg_sig([(7, M[0]), (7, M[1]), (8, M[2]), (9, M[2])])),
    ]
    want = [int(B.AggregateVerify(p, m, s)) for _, p, m, s in sets]
    assert want == [1, 0, 1, 0, 0, 0, 1]
    got = _run([s[1:] for s in sets])
    assert got == want, [(n, g, w) for (n, *_), g, w in zip(sets, got, want) if g != w]


def test_aggregate_verify_core_set_boundaries():
    """The set of an item is found by binary search in the offsets: leading, trailing and consecutive empty sets, and a set whose
    signature belongs to its neighbour"""
    a = [(0, M[0]), (1, M[1])]
    b = [(2, M[2])]
    sa, sb = _agg_sig(a), _agg_sig(b)
    pa, ma = [_pk(k) for k, _ in a], [m for _, m in a]
    pb, mb = [_pk(k) for k, _ in b], [m for _, m in b]
    sets = [([], [], sa), (pa, ma, sa), ([], [], sb), ([], [], sb), (pb, mb, sb), (pb, mb, sa), ([], [], sa)]
    assert _run(sets) == [0, 1, 0, 0, 1, 0, 0]
