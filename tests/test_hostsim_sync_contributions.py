"""The __host__ __device__ SSZ roots and aggregator selection of csrc/synccontrib.cuh, compiled with g++ (tests/hostsim/synccontrib_sim.cpp),
against tests/sync_contributions_oracle.py: the Bitvector root at one to four chunks, the SyncCommitteeContribution and ContributionAndProof
roots, the three signing roots and is_sync_committee_aggregator at several targets."""
import ctypes
import os
import shutil
import subprocess
import tempfile

import numpy as np

import hs
import sync_contributions_oracle as C


def _build():
    """g++ build of tests/hostsim/synccontrib_sim.cpp in a temporary directory: the tree is not written"""
    root = os.path.dirname(hs.HERE)
    d = tempfile.mkdtemp(prefix="synccontrib_sim_")
    try:
        out = os.path.join(d, "libsynccontrib_sim.so")
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-x", "c++", "-I", os.path.join(root, "pos_evolution_b200", "csrc"),
                               os.path.join(hs.HERE, "hostsim", "synccontrib_sim.cpp"), "-o", out])
        return ctypes.CDLL(out)
    finally:
        shutil.rmtree(d, ignore_errors=True)      # the loaded library stays mapped


def test_hostsim_roots_match_oracle():
    lib = _build()
    rng = np.random.default_rng(17)
    doms = [rng.bytes(32) for _ in range(3)]
    for sub in (1, 3, 8, 128, 255, 256, 257, 600, 768, 1024):
        sb = (sub + 7) // 8
        items = []
        for _ in range(6):
            bits = [bool(x) for x in rng.integers(0, 2, sub)]
            items.append(C.encode(int(rng.integers(0, 2**63)), int(rng.integers(0, 2**63)), rng.bytes(32), int(rng.integers(0, 2**63)), bits,
                                  rng.bytes(96), rng.bytes(96), rng.bytes(96)))
        n = len(items)
        wire = np.frombuffer(b"".join(items), np.uint8).copy()
        outs = [np.zeros((n, 32), np.uint8) for _ in range(6)]
        d = [np.frombuffer(x, np.uint8).copy() for x in doms]
        lib.hs_sync_contribution_roots(hs.ptr(wire), ctypes.c_uint32(sb), ctypes.c_uint64(n), hs.ptr(d[0]), hs.ptr(d[1]), hs.ptr(d[2]),
                                       *[hs.ptr(o) for o in outs])
        for i, w in enumerate(items):
            g, slot, root, s, row, sig, proof, outer = C.decode(w, sb)
            assert outs[0][i].tobytes() == C.bitvector_root(row), (sub, i)
            assert outs[1][i].tobytes() == C.contribution_root(slot, root, s, row, sig), (sub, i)
            cap = C.contribution_and_proof_root(g, slot, root, s, row, sig, proof)
            assert outs[2][i].tobytes() == cap, (sub, i)
            assert outs[3][i].tobytes() == C.signing_root(C.selection_data_root(slot, s), doms[1]), (sub, i)
            assert outs[4][i].tobytes() == C.signing_root(cap, doms[2]), (sub, i)
            assert outs[5][i].tobytes() == C.signing_root(root, doms[0]), (sub, i)


def test_hostsim_is_aggregator_matches_oracle():
    lib = _build()
    rng = np.random.default_rng(18)
    n = 400
    subs = np.array(rng.integers(1, 1025, n), np.uint32)
    subs[:4] = [8, 128, 16, 1]
    pr = np.frombuffer(rng.bytes(96 * n), np.uint8).copy()
    for target in (16, 4, 1, 2000):
        out = np.zeros(n, np.uint8)
        lib.hs_sync_is_aggregator(hs.ptr(pr), hs.ptr(subs), ctypes.c_uint32(target), ctypes.c_uint64(n), hs.ptr(out))
        want = [int(C.is_aggregator(pr[96 * i:96 * i + 96].tobytes(), int(subs[i]), target)) for i in range(n)]
        assert out.tolist() == want, target
        if target == 1:
            assert 0 < sum(want) < n
