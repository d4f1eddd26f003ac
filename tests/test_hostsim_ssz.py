"""The node hash and the Validator leaf of csrc/ssz.cuh on the CPU (tests/hostsim/ssz_sim.cpp) against hashlib and the SSZ oracle."""
import ctypes
import hashlib
import os
import shutil
import subprocess
import tempfile

import numpy as np

import hs
import ssz_oracle as O
from pos_evolution_b200 import spec as PS


def _build():
    """g++ build of tests/hostsim/ssz_sim.cpp in a temporary directory: the tree is not written"""
    root = os.path.dirname(hs.HERE)
    d = tempfile.mkdtemp(prefix="ssz_sim_")
    try:
        out = os.path.join(d, "libssz_sim.so")
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-x", "c++", "-I", os.path.join(root, "pos_evolution_b200", "csrc"),
                               os.path.join(hs.HERE, "hostsim", "ssz_sim.cpp"), "-o", out])
        return ctypes.CDLL(out)
    finally:
        shutil.rmtree(d, ignore_errors=True)      # the loaded library stays mapped


lib = _build()


def _node_digests(nodes: bytes) -> bytes:
    """64-byte nodes -> their SHA-256 through hs_sha256_node, converting bytes to and from digest-word order"""
    n = len(nodes) // 64
    words = np.frombuffer(nodes, dtype=">u4").astype(np.uint32)
    out = np.zeros(8 * n, dtype=np.uint32)
    lib.hs_sha256_node(hs.ptr(words), ctypes.c_uint64(n), hs.ptr(out))
    return out.astype(">u4").tobytes()


def test_sha256_node_matches_hashlib():
    rng = np.random.default_rng(1)
    nodes = [bytes(64), b"\xff" * 64, bytes(range(64))] + [rng.bytes(64) for _ in range(200)]
    got = _node_digests(b"".join(nodes))
    for i, m in enumerate(nodes):
        assert got[32 * i:32 * i + 32] == hashlib.sha256(m).digest(), i
    assert got[:32] == O.ZERO_HASHES[1]


def _random_validator(rng):
    far = PS.FAR_FUTURE_EPOCH
    pick = lambda: [0, 1, 2**32 - 1, 2**32, far, int(rng.integers(0, 2**63))][int(rng.integers(0, 6))]      # noqa: E731
    return PS.Validator(rng.bytes(48), int(rng.integers(0, 2**63)), bool(rng.integers(0, 2)), pick(), pick(), withdrawal_credentials=rng.bytes(32),
                        activation_eligibility_epoch=pick(), withdrawable_epoch=pick())


def test_validator_leaf_matches_oracle():
    rng = np.random.default_rng(2)
    vals = [_random_validator(rng) for _ in range(300)]
    vals.append(PS.Validator(bytes(48), 0))
    vals.append(PS.Validator(b"\xff" * 48, 2**64 - 1, True, 2**64 - 1, 2**64 - 1, b"\xff" * 32, 2**64 - 1, 2**64 - 1))
    rec = PS.serialize_validators(vals)
    assert [bytes(r) for r in rec] == [O.serialize_validator(v) for v in vals]
    out = np.zeros((len(vals), 32), dtype=np.uint8)
    lib.hs_validator_root(hs.ptr(rec), ctypes.c_uint64(len(vals)), hs.ptr(out))
    for i, v in enumerate(vals):
        assert bytes(out[i]) == O.validator_root(v), i
