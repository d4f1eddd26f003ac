"""The SSZ merkleization rules of tests/ssz_oracle.py on hand-built cases (CPU only)."""
import hashlib

import pytest

import ssz_oracle as O
from oracle import ssz as lite
from pos_evolution_b200 import spec as PS


def H(a, b):
    return hashlib.sha256(a + b).digest()


def _naive(chunks, width):
    """the full tree: chunks padded with explicit zero chunks to `width`"""
    layer = list(chunks) + [bytes(32)] * (width - len(chunks))
    while len(layer) > 1:
        layer = [H(layer[i], layer[i + 1]) for i in range(0, len(layer), 2)]
    return layer[0]


def test_zero_hash_chain():
    assert O.ZERO_HASHES[0] == bytes(32)
    assert O.ZERO_HASHES[1].hex() == "f5a5fd42d16a20302798ef6ed309979b43003d2320d9f0e8ea9831a92759fb4b"
    for l in range(1, 10):
        assert O.ZERO_HASHES[l] == _naive([], 1 << l)


@pytest.mark.parametrize("log_limit", range(13))
def test_virtual_limit_equals_zero_padding(log_limit):
    limit = 1 << log_limit
    counts = sorted({0, 1, 2, 3, limit // 2, limit // 2 + 1, limit - 1, limit} & set(range(limit + 1)))
    for n in counts:
        chunks = [hashlib.sha256(b"chunk%d" % i).digest() for i in range(n)]
        assert O.merkleize(chunks, limit) == _naive(chunks, limit), n
        # a limit that is not a power of two pads to the next one
        if limit > 2 and n <= limit - 1:
            assert O.merkleize(chunks, limit - 1) == _naive(chunks, limit)


def test_list_rules():
    r = [hashlib.sha256(b"r%d" % i).digest() for i in range(9)]
    ln = lambda k: k.to_bytes(32, "little")      # noqa: E731
    # List[Root, 16]: empty, one element, a power of two, one past it
    assert O.roots_list_root([], 16) == H(O.ZERO_HASHES[4], ln(0))
    assert O.roots_list_root(r[:1], 16) == H(H(H(H(H(r[0], O.ZERO_HASHES[0]), O.ZERO_HASHES[1]), O.ZERO_HASHES[2]), O.ZERO_HASHES[3]), ln(1))
    four = H(H(r[0], r[1]), H(r[2], r[3]))
    assert O.roots_list_root(r[:4], 16) == H(H(H(four, O.ZERO_HASHES[2]), O.ZERO_HASHES[3]), ln(4))
    five = H(four, H(H(r[4], bytes(32)), O.ZERO_HASHES[1]))
    assert O.roots_list_root(r[:5], 16) == H(H(five, O.ZERO_HASHES[3]), ln(5))
    # List[uint64, 2^40]: four values share one chunk; the tree has 2^38 chunks
    chunk = b"".join(v.to_bytes(8, "little") for v in (1, 2, 3, 4))
    assert O.basic_list_root([1, 2, 3, 4], 8, 2**40) == H(_chain(chunk, 0, 38), ln(4))
    assert O.basic_list_root([], 8, 2**40) == H(O.ZERO_HASHES[38], ln(0))
    assert O.basic_list_root([7], 1, 2**40) == H(_chain(bytes([7]) + bytes(31), 0, 35), ln(1))
    # Vector[uint64, 5]: two chunks
    assert O.basic_vector_root([1, 2, 3, 4, 5], 8) == H(chunk, (5).to_bytes(8, "little") + bytes(24))
    # ByteList[32] of 3 bytes, Bitvector[4]
    assert O.byte_list_root(b"abc", 32) == H(b"abc" + bytes(29), ln(3))
    assert O.bitvector_root([1, 0, 1, 1]) == bytes([0b1101]) + bytes(31)


def _chain(node, lo, hi):
    """node padded with zero subtrees from depth lo to depth hi"""
    for l in range(lo, hi):
        node = H(node, O.ZERO_HASHES[l])
    return node


def test_container_rules():
    cp = PS.Checkpoint(7, hashlib.sha256(b"cp").digest())
    assert O.checkpoint_root(cp) == lite.htr_checkpoint(cp.epoch, cp.root) == PS.hash_tree_root_checkpoint(cp)
    pk = bytes(range(48))
    assert O.pubkey_root(pk) == H(pk[:32], pk[32:] + bytes(16))
    v = PS.Validator(pk, 32 * 10**9, True, 5, 9, withdrawal_credentials=b"\x01" * 32, activation_eligibility_epoch=4, withdrawable_epoch=300)
    u = lambda x: x.to_bytes(8, "little") + bytes(24)      # noqa: E731
    leaves = [O.pubkey_root(pk), b"\x01" * 32, u(32 * 10**9), b"\x01" + bytes(31), u(4), u(5), u(9), u(300)]
    assert O.validator_root(v) == _naive(leaves, 8)
    assert O.validators_root([v], 2**40) == H(_chain(O.validator_root(v), 0, 40), (1).to_bytes(32, "little"))
    f = PS.Fork(b"\x00\x00\x00\x01", b"\x00\x00\x00\x02", 3)
    assert O.fork_root(f) == _naive([b"\x00\x00\x00\x01" + bytes(28), b"\x00\x00\x00\x02" + bytes(28), u(3)], 4)
    hdr = PS.ExecutionPayloadHeader(extra_data=b"xy", base_fee_per_gas=2**200)
    root = O.execution_payload_header_root(hdr)
    leaves = [bytes(32)] * 4 + [O.ZERO_HASHES[3], bytes(32)] + [bytes(32)] * 4 + [H(b"xy" + bytes(30), (2).to_bytes(32, "little")),
                                                                                 (2**200).to_bytes(32, "little"), bytes(32), bytes(32)]
    assert root == _naive(leaves, 16)


def test_sparse_list_root_equals_full_tree():
    dflt = hashlib.sha256(b"leaf").digest()
    for n in (1, 5, 8, 13, 64):
        over = {i: hashlib.sha256(b"o%d" % i).digest() for i in (0, n // 2, n - 1)}
        leaves = [over.get(i, dflt) for i in range(n)]
        assert O.sparse_list_root(n, dflt, over, 2**10) == O.mix_in_length(O.merkleize(leaves, 2**10), n)
