"""The aggregated-attestation intake on the CPU: the oracle's roots and aggregator selection against hashlib and the SSZ oracle, the
host-compiled root code of csrc/aggintake.cuh (tests/hostsim/aggintake_sim.cpp) against the oracle, the list-order semantics of checks 10
and 11 on hand-built cases, and Spec.validate_aggregate_and_proofs' split by epoch with a stub engine."""
import ctypes
import hashlib
import os
import shutil
import subprocess
import tempfile

import numpy as np
import pytest

import aggregate_intake_oracle as A
import hs
import ssz_oracle as S
from intake_oracle import data128 as make_data
from oracle.spec import AttestationData, Checkpoint, hash_tree_root_attestation_data
from pos_evolution_b200 import spec as PS


def _build():
    """g++ build of tests/hostsim/aggintake_sim.cpp in a temporary directory: the tree is not written"""
    root = os.path.dirname(hs.HERE)
    d = tempfile.mkdtemp(prefix="aggintake_sim_")
    try:
        out = os.path.join(d, "libaggintake_sim.so")
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-x", "c++", "-I", os.path.join(root, "pos_evolution_b200", "csrc"),
                               os.path.join(hs.HERE, "hostsim", "aggintake_sim.cpp"), "-o", out])
        return ctypes.CDLL(out)
    finally:
        shutil.rmtree(d, ignore_errors=True)      # the loaded library stays mapped


def _random_item(rng, nbits):
    bits = [bool(x) for x in rng.integers(0, 2, nbits)]
    d = make_data(int(rng.integers(0, 2**40)), int(rng.integers(0, 64)), rng.bytes(32), int(rng.integers(0, 2**30)), rng.bytes(32),
                  int(rng.integers(0, 2**30)), rng.bytes(32))
    return int(rng.integers(0, 2**63)), bits, d, rng.bytes(96), rng.bytes(96)


def test_oracle_roots_against_ssz_oracle():
    rng = np.random.default_rng(3)
    for nbits in (1, 7, 8, 31, 256, 511, 512, 2047, 2048):
        agg, bits, d, sig, proof = _random_item(rng, nbits)
        # Bitlist[2048]: the packed bits in 8 chunks, mixed with the length
        packed = bytes(sum(1 << k for k in range(8) if j + k < nbits and bits[j + k]) for j in range(0, nbits, 8))
        chunks = [packed[i:i + 32].ljust(32, b"\0") for i in range(0, 256, 32)]
        while len(chunks) > 1:
            chunks = [hashlib.sha256(chunks[i] + chunks[i + 1]).digest() for i in range(0, len(chunks), 2)]
        assert A.bitlist_root(bits) == hashlib.sha256(chunks[0] + nbits.to_bytes(32, "little")).digest()
        dd = AttestationData(int.from_bytes(d[0:8], "little"), int.from_bytes(d[8:16], "little"), d[16:48],
                             Checkpoint(int.from_bytes(d[48:56], "little"), d[56:88]), Checkpoint(int.from_bytes(d[88:96], "little"), d[96:128]))
        assert A.data_root(d) == hash_tree_root_attestation_data(dd)
        h = lambda x, y: hashlib.sha256(x + y).digest()      # noqa: E731
        sr = lambda s: h(h(s[0:32], s[32:64]), h(s[64:96], bytes(32)))      # noqa: E731
        att = h(h(A.bitlist_root(bits), A.data_root(d)), h(sr(sig), bytes(32)))
        assert A.signature_root(sig) == sr(sig) and A.attestation_root(bits, d, sig) == att
        assert A.aggregate_and_proof_root(agg, bits, d, sig, proof) == h(h(S.uint_root(agg), att), h(sr(proof), bytes(32)))
        dom = rng.bytes(32)
        assert A.slot_signing_root(12345, dom) == h((12345).to_bytes(32, "little"), dom)


def test_oracle_is_aggregator():
    rng = np.random.default_rng(4)
    for size in (1, 15, 16, 31, 32, 47, 512, 2048):
        for _ in range(20):
            proof = rng.bytes(96)
            v = int.from_bytes(hashlib.sha256(proof).digest()[:8], "little")
            assert A.is_aggregator(size, proof) == (v % max(1, size // 16) == 0)
    assert all(A.is_aggregator(15, rng.bytes(96)) for _ in range(10))      # modulo 1: every member is an aggregator


def test_hostsim_roots_match_oracle():
    lib = _build()
    rng = np.random.default_rng(5)
    stride = 256
    items = [_random_item(rng, int(nb)) for nb in [1, 8, 9, 100, 255, 256, 512, 1000, 2047, 2048] + list(rng.integers(1, 2049, 30))]
    n = len(items)
    aggs = np.array([x[0] for x in items], np.uint64)
    rows = np.zeros((n, stride), np.uint8)
    nbits = np.array([len(x[1]) for x in items], np.uint32)
    for i, x in enumerate(items):
        for j, b in enumerate(x[1]):
            if b:
                rows[i, j >> 3] |= 1 << (j & 7)
    data = np.frombuffer(b"".join(x[2] for x in items), np.uint8).copy()
    sigs = np.frombuffer(b"".join(x[3] for x in items), np.uint8).copy()
    proofs = np.frombuffer(b"".join(x[4] for x in items), np.uint8).copy()
    dsel, daap = np.frombuffer(rng.bytes(32), np.uint8).copy(), np.frombuffer(rng.bytes(32), np.uint8).copy()
    root, slot_root, aap_sr = (np.zeros((n, 32), np.uint8) for _ in range(3))
    lib.hs_aggregate_and_proof_roots(hs.ptr(aggs), hs.ptr(rows), ctypes.c_uint32(stride), hs.ptr(nbits), hs.ptr(data), hs.ptr(sigs), hs.ptr(proofs),
                                     hs.ptr(dsel), hs.ptr(daap), ctypes.c_uint64(n), hs.ptr(root), hs.ptr(slot_root), hs.ptr(aap_sr))
    for i, (agg, bits, d, sig, proof) in enumerate(items):
        assert root[i].tobytes() == A.aggregate_and_proof_root(agg, bits, d, sig, proof), i
        assert aap_sr[i].tobytes() == A.aggregate_and_proof_signing_root(agg, bits, d, sig, proof, daap.tobytes()), i
        assert slot_root[i].tobytes() == A.slot_signing_root(int.from_bytes(d[0:8], "little"), dsel.tobytes()), i
    sizes = np.array(rng.integers(1, 2049, 300), np.uint32)
    pr = np.frombuffer(rng.bytes(96 * 300), np.uint8).copy()
    for target in (16, 8, 1):
        out = np.zeros(300, np.uint8)
        lib.hs_is_aggregator(hs.ptr(pr), hs.ptr(sizes), ctypes.c_uint32(target), ctypes.c_uint64(300), hs.ptr(out))
        assert out.tolist() == [int(A.is_aggregator(int(sizes[i]), pr[96 * i:96 * i + 96].tobytes(), target)) for i in range(300)]


# ------------------------------------------------------------------------------------------ list-order semantics (checks 10 and 11)
SPE, CPS, STRIDE = 4, 2, 4


def _setup():
    """epoch 1 of 4 slots x 2 committees of 8 members (validators 0..63); a tree of one block at slot 0 that every item votes for"""
    members = np.arange(64, dtype=np.uint32)
    off = np.arange(9, dtype=np.uint32) * 8
    parent, slot, roots = np.zeros(1, np.uint32), np.zeros(1, np.uint64), np.full((1, 32), 7, np.uint8)
    return members, off, parent, slot, roots


def _item(c, bits, agg, head=b"\x07" * 32):
    s, idx = 4 + c // CPS, c % CPS
    d = make_data(s, idx, head, 0, b"\x07" * 32, 1, b"\x07" * 32)
    return A.encode(agg, bits, d, bytes([c]) * 96, bytes(96), bytes(96))


def _run(wires, bad=()):
    members, off, parent, slot, roots = _setup()
    ok = lambda i: (True, True, i not in bad)      # noqa: E731
    return A.validate(wires, members, off, 1, 7, bytes(96), CPS, SPE, STRIDE, parent, slot, roots, ok, target=16).status.tolist()


def test_list_order_duplicates_and_subsets():
    full, half, other = [True] * 8, [True] * 4 + [False] * 4, [False] * 4 + [True] * 4
    # an earlier duplicate that fails a signature check does not shadow a later valid one
    assert _run([_item(0, full, 0), _item(0, full, 1)], bad={0}) == [16, 0]
    # a subset after its superset is ignored (10), also when byte-equal; a superset after its subset is accepted
    assert _run([_item(0, full, 0), _item(0, half, 1), _item(0, full, 2)]) == [0, 10, 10]
    assert _run([_item(0, half, 0), _item(0, full, 1)]) == [0, 0]
    # disjoint bits of the same data are both accepted; the same aggregator again is 11
    assert _run([_item(0, half, 0), _item(0, other, 1), _item(0, full[:7] + [False], 0)]) == [0, 0, 11]
    # 11 needs an ACCEPTED earlier item: a failed one does not count
    assert _run([_item(0, full, 2), _item(0, half, 2)], bad={0}) == [16, 0]
    # an aggregator from another committee: 11 once that aggregator was accepted earlier, 13 otherwise
    assert _run([_item(1, full, 9), _item(0, full, 9)]) == [0, 11]
    assert _run([_item(0, full, 9), _item(1, full, 9)]) == [13, 0]
    # different data of one committee do not shadow each other
    assert _run([_item(0, full, 0), _item(0, half, 1, head=b"\x08" * 32)]) == [0, 17]


# ------------------------------------------------------------------------------------------ the facade's split by epoch
class _StubEngine:
    def __init__(self):
        self.calls = []

    def aggregate_and_proof_intake(self, wire, woff, members, off, epoch, current_slot, domains96, cps, spe, stride, target, prop_range):
        n = len(woff) - 1
        self.calls.append((epoch, n, current_slot, len(domains96), stride, target, prop_range))
        return type("R", (), {"status": np.full(n, 0 if epoch % 2 else 16, np.int32)})()


def test_facade_splits_by_epoch(monkeypatch):
    stub = _StubEngine()
    sp = PS.Spec(PS.MINIMAL, engine=stub, incremental_tree=True)
    monkeypatch.setattr(sp, "_sync_store", lambda store: None)
    monkeypatch.setattr(sp, "sync_registry", lambda state: None)
    monkeypatch.setattr(sp, "epoch_committees", lambda state, epoch: (np.arange(8, dtype=np.uint32), np.array([0, 8], np.uint32), 1))
    monkeypatch.setattr(sp, "get_domain", lambda state, d, epoch: bytes(d) + bytes(28))

    def item(slot):
        data = PS.AttestationData(slot, 0, bytes(32), PS.Checkpoint(0, bytes(32)), PS.Checkpoint(slot // 8, bytes(32)))
        return PS.SignedAggregateAndProof(PS.AggregateAndProof(3, PS.Attestation([True] * 8, data, bytes(96)), bytes(96)), bytes(96))

    items = [item(s) for s in (25, 17, 3, 30, 40, 16, 31)]      # epochs 3, 2, 0, 3, 5, 2, 3 (minimal: 8 slots per epoch)
    status, accepted = sp.validate_aggregate_and_proofs(None, None, items, current_slot=26)
    assert stub.calls == [(3, 3, 26, 96, 1, 16, 32), (2, 2, 26, 96, 1, 16, 32)]
    assert status == [0, 16, 7, 0, 7, 16, 0]
    assert accepted == [items[0].message.aggregate, items[3].message.aggregate, items[6].message.aggregate]
    wire = PS.serialize_signed_aggregate_and_proof(items[0])
    assert len(wire) == 100 + 108 + 228 + 2 and wire == A.encode(3, [True] * 8, PS.serialize_attestation_data(items[0].message.aggregate.data),
                                                                  bytes(96), bytes(96), bytes(96))
    with pytest.raises(ValueError):
        PS.Spec(PS.MINIMAL, engine=stub).validate_aggregate_and_proofs(None, None, items, current_slot=26)
