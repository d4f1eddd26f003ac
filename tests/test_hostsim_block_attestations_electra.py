"""The __host__ __device__ decode and checks 1-12 of csrc/blockatt_electra.cuh, compiled with g++ (tests/hostsim/blockatt_electra_sim.cpp),
against tests/block_attestations_electra_oracle.py over random and adversarial encodings: wrong offsets, truncation, a committee_bits padding
bit, Bitlists at the limit and one past it, empty and misplaced committee segments, and the lane-split bit scan the kernel runs."""
import ctypes
import os
import shutil
import subprocess
import tempfile

import numpy as np
import pytest

import block_attestations_electra_oracle as E
import hs
from oracle.spec import integer_squareroot


def _build():
    """g++ build of tests/hostsim/blockatt_electra_sim.cpp in a temporary directory: the tree is not written"""
    root = os.path.dirname(hs.HERE)
    d = tempfile.mkdtemp(prefix="blockatt_electra_sim_")
    try:
        out = os.path.join(d, "libblockatt_electra_sim.so")
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-x", "c++", "-I", os.path.join(root, "pos_evolution_b200", "csrc"),
                               os.path.join(hs.HERE, "hostsim", "blockatt_electra_sim.cpp"), "-o", out])
        return ctypes.CDLL(out)
    finally:
        shutil.rmtree(d, ignore_errors=True)      # the loaded library stays mapped


@pytest.fixture(scope="module")
def lib():
    return _build()


class Layout:
    """committees of epochs e - 1 and e with random sizes; the chain's roots and justified checkpoints"""

    def __init__(self, rng, M, max_vpc, spe, e, cps_prev, cps_cur):
        self.M, self.max_vpc, self.spe, self.e, self.cps_prev, self.cps_cur = M, max_vpc, spe, e, cps_prev, cps_cur
        sizes = rng.integers(0, max_vpc + 1, (cps_prev + cps_cur) * spe)
        sizes = np.where(rng.random(sizes.size) < 0.9, np.maximum(sizes, 1), sizes)      # a few empty committees
        self.off = np.concatenate([[0], np.cumsum(sizes)]).astype(np.uint32)
        self.members = rng.permutation(int(self.off[-1]) + 7)[:int(self.off[-1])].astype(np.uint32)
        self.roots = [bytes(rng.integers(0, 256, 32, dtype=np.uint8)) for _ in range(2 * spe)]
        self.justified = bytes(rng.integers(0, 256, 80, dtype=np.uint8))

    def size(self, slot, ci):
        E_ = slot // self.spe
        cur = E_ == self.e
        cps = self.cps_cur if cur else self.cps_prev
        c = (self.cps_prev * self.spe if cur else 0) + (slot - E_ * self.spe) * cps + ci
        return int(self.off[c + 1] - self.off[c])

    def att(self, rng, block_slot):
        """a random attestation, right more often than not, then perhaps one mutation"""
        lo = max((self.e - 1) * self.spe, 0)
        slot = int(rng.integers(lo, block_slot)) if rng.random() < 0.9 else int(rng.integers(lo, (self.e + 1) * self.spe))
        E_ = slot // self.spe
        cps = self.cps_cur if E_ == self.e else self.cps_prev
        picks = [i for i in range(min(cps, self.M)) if rng.random() < 0.5] or [0]
        if rng.random() < 0.1:
            picks = sorted(set(picks + [int(rng.integers(0, self.M))]))      # perhaps an index >= committees_per_slot
        bits = []
        for ci in picks:
            n = self.size(slot, ci) if ci < cps else int(rng.integers(0, 4))
            row = [bool(x) for x in rng.random(n) < 0.6]
            if rng.random() < 0.1:
                row = [False] * n
            bits += row
        if rng.random() < 0.1 and bits:
            bits = bits[:-1] if rng.random() < 0.5 else bits + [True]
        cur = E_ == self.e
        src = self.justified[40:80] if cur else self.justified[0:40]
        if rng.random() < 0.05:
            src = bytes(40)
        head = self.roots[slot + self.spe - self.e * self.spe] if rng.random() < 0.7 else bytes(32)
        troot = self.roots[self.spe if cur else 0] if rng.random() < 0.8 else bytes(32)
        tepoch = E_ if rng.random() < 0.95 else int(rng.integers(0, self.e + 2))
        index = 0 if rng.random() < 0.95 else int(rng.integers(1, 3))
        d = E.data128(slot, index, head, int.from_bytes(src[:8], "little"), src[8:], tepoch, troot)
        w = bytearray(E.encode(bits, d, bytes(rng.integers(0, 256, 96, dtype=np.uint8)), E.committee_bits_of(picks, self.M)))
        r = rng.random()
        F = E.fixed(self.M)
        if r < 0.04:
            w = w[:int(rng.integers(0, len(w)))]                                    # truncated
        elif r < 0.07:
            w[0:4] = (F + int(rng.choice([-1, 1, 4]))).to_bytes(4, "little")       # a wrong offset
        elif r < 0.10 and self.M % 8:
            w[F - 1] |= 1 << int(rng.integers(self.M % 8, 8))                       # a padding bit of committee_bits
        elif r < 0.12:
            w = w[:F]                                                                # no Bitlist byte
        elif r < 0.14:
            w[-1] = 0                                                                # no delimiter
        elif r < 0.16:
            w = bytes(w[:F]) + E.bitlist([True] * (self.max_vpc * self.M + int(rng.integers(0, 2))))     # the limit and one past it
        return bytes(w)

    def host(self, lib, wires, bslots):
        woff = np.concatenate([[0], np.cumsum([len(w) for w in wires])]).astype(np.uint32)
        wire = np.frombuffer(b"".join(wires) + bytes(1), np.uint8).copy()
        n = len(wires)
        st, mask, nb, cm = np.zeros(n, np.int32), np.zeros(n, np.uint8), np.zeros(n, np.uint32), np.zeros(n, np.uint64)
        roots = np.frombuffer(b"".join(self.roots), np.uint8).copy()
        j = np.frombuffer(self.justified, np.uint8).copy()
        bs = np.asarray(bslots, np.uint64)
        row_max = E.row_max(self.off, self.cps_prev, self.cps_cur, self.spe)
        lib.hs_bae_check(hs.ptr(wire), hs.ptr(woff), ctypes.c_uint32(n), hs.ptr(bs), ctypes.c_uint64(self.e), hs.ptr(self.off),
                         ctypes.c_uint64(len(self.members)), ctypes.c_uint32(self.M), ctypes.c_uint32(self.max_vpc), ctypes.c_uint32(self.cps_prev),
                         ctypes.c_uint32(self.cps_cur), ctypes.c_uint32(self.spe), ctypes.c_uint32(1), ctypes.c_uint32(integer_squareroot(self.spe)),
                         ctypes.c_uint32(row_max), hs.ptr(roots), hs.ptr(j), hs.ptr(st), hs.ptr(mask), hs.ptr(nb), hs.ptr(cm))
        return st, mask, nb, cm

    def oracle(self, w, bslot):
        return E.check(w, bslot, self.e, self.members, self.off, self.cps_prev, self.cps_cur, self.roots, self.justified, bytes(64), self.spe, 1,
                       self.M, self.max_vpc, lambda *a: True)


@pytest.mark.parametrize("M,max_vpc,spe,cps_prev,cps_cur,seed", [(4, 9, 8, 2, 4, 1), (6, 12, 4, 4, 5, 2), (64, 5, 4, 40, 64, 3), (1, 30, 8, 1, 1, 4),
                                                                   (9, 7, 2, 3, 9, 5)])
def test_hostsim_checks_match_oracle(lib, M, max_vpc, spe, cps_prev, cps_cur, seed):
    rng = np.random.default_rng(seed)
    L = Layout(rng, M, max_vpc, spe, 3, cps_prev, cps_cur)
    wires, bslots = [], []
    for _ in range(1500):
        bslot = int(rng.integers(3 * spe, 4 * spe))
        wires.append(L.att(rng, bslot))
        bslots.append(bslot)
    st, mask, nb, cm = L.host(lib, wires, bslots)
    seen = set()
    for i, (w, b) in enumerate(zip(wires, bslots)):
        o_st, o_mask, _, _ = L.oracle(w, b)
        assert (int(st[i]), int(mask[i])) == (o_st, o_mask), (i, w.hex())
        seen.add(o_st)
        if o_st == 0:
            _, bits, cbits = E.decode(w, M, max_vpc * M)
            assert int(nb[i]) == len(bits) and int(cm[i]) == sum(1 << k for k, x in enumerate(cbits) if x)
    assert seen >= {0, 1, 2, 4, 5, 6, 7, 10} | ({8} if cps_cur < M else set())


def test_hostsim_every_status_and_the_limit(lib):
    """one hand-made attestation per status 0-12 on the minimal shape (M = 4), and Bitlists of exactly the limit and one more"""
    rng = np.random.default_rng(9)
    L = Layout(rng, 4, 6, 8, 3, 2, 3)
    L.off = np.arange(0, 6 * 5 * 8 + 1, 6, dtype=np.uint32)[:5 * 8 + 1]      # every committee 6 members
    L.members = np.arange(int(L.off[-1]), dtype=np.uint32)
    s = 28
    cur = L.justified[40:80]

    def a(slot, picks, bits=None, index=0, src=cur, tepoch=None, M=4):
        tepoch = slot // 8 if tepoch is None else tepoch
        bits = [True] * (6 * len(picks)) if bits is None else bits
        d = E.data128(slot, index, L.roots[slot + 8 - 24], int.from_bytes(src[:8], "little"), src[8:], tepoch, L.roots[8 if tepoch == 3 else 0])
        return E.encode(bits, d, bytes(96), E.committee_bits_of(picks, M))

    good = a(27, [0, 2])
    F = E.fixed(4)
    cases = [(good, 0), (good[:100], 1), (bytes([F + 1]) + good[1:], 1), (good[:F - 1] + bytes([good[F - 1] | 0x10]) + good[F:], 1),
             (good[:F], 2), (good[:-1] + bytes(1), 2), (good[:F] + E.bitlist([True] * 25), 3), (good[:F] + E.bitlist([True] * 24), 10),
             (a(12, [0], tepoch=1), 4), (a(20, [0], tepoch=3), 5), (a(28, [0]), 6), (a(27, [0], index=1), 7), (a(27, [0, 3]), 8),
             (a(27, [1, 2], bits=[True] * 6 + [False] * 6), 9), (a(27, [1, 2], bits=[True] * 11), 10), (a(27, [1], bits=[True] * 7), 10),
             (a(27, [0], src=L.justified[0:40]), 11), (a(27, []), 12), (a(27, [], bits=[True]), 10), (a(20, [1], tepoch=2, src=L.justified[0:40]), 0)]
    L.cps_prev, L.cps_cur = 2, 3
    wires = [w for w, _ in cases]
    st, mask, _, _ = L.host(lib, wires, [s] * len(wires))
    assert st.tolist() == [x for _, x in cases]
    assert [L.oracle(w, s)[0] for w in wires] == [x for _, x in cases]
    assert mask[0] == 7 and mask[-1] == 2        # delay 1 on the head; delay 8 > isqrt: target only (no upper bound since Deneb)


def test_hostsim_lane_split_bit_scan(lib):
    """bae_any_bit spread over 1, 3 and 32 lanes against a direct scan, on every [lo, hi) of a sparse 40-byte row"""
    rng = np.random.default_rng(11)
    for trial in range(20):
        row = np.zeros(40, np.uint8)
        for _ in range(int(rng.integers(0, 3))):
            k = int(rng.integers(0, 320))
            row[k >> 3] |= 1 << (k & 7)
        bits = [(row[k >> 3] >> (k & 7)) & 1 for k in range(320)]
        for lo in range(0, 320, 7 + trial):
            for hi in range(lo, 321, 5 + trial):
                want = int(any(bits[lo:hi]))
                for nl in (1, 3, 32):
                    assert lib.hs_bae_any_bit(hs.ptr(row), ctypes.c_uint32(lo), ctypes.c_uint32(hi), ctypes.c_uint32(nl)) == want
