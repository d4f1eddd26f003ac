"""Adversarial keys for the two device intakes (csrc/intake.cuh, csrc/aggintake.cuh): AttestationData that share the 32-bit fingerprint
the kernels compare before the 128 data bytes, and block roots that differ from each other, or from a tree root, in one byte only.

The fingerprint XORs one bijection per 4-byte word k of the data (lane k of the warp): x = (w ^ k * LANE_KEY) * MIX, then x ^ (x >> 15),
all mod 2^32.  Each lane inverts, so rewriting one word sets the fingerprint to any value.  The free words are the source checkpoint
(data bytes 48..87, words 12..21): neither intake reads it, so data that differ there pass every check.  Words 4..11 (the head root)
and 24..31 (the target root) are rewritten only where a test wants that field to differ.  test_intake_keys.py pins this restatement to
the source text of both kernels."""
import numpy as np

LANE_KEY, MIX = 0x9E3779B9, 0x85EBCA6B
M32 = 0xFFFFFFFF
_MIX_INV = pow(MIX, -1, 1 << 32)
FREE_LANES = tuple(range(12, 22))
HEAD_LANES, TARGET_LANES = tuple(range(4, 12)), tuple(range(24, 32))
OUTSIDE = b"\xff" * 32                     # intake_oracle.block_store's parent of the root block: never a tree root


def _word(d, k):
    return int.from_bytes(d[4 * k:4 * k + 4], "little")


def _set_word(d, k, w):
    d = bytearray(d)
    d[4 * k:4 * k + 4] = (w & M32).to_bytes(4, "little")
    return bytes(d)


def lane(w, k):
    """lane k's mix of data word w"""
    x = ((w ^ (k * LANE_KEY & M32)) * MIX) & M32
    return x ^ (x >> 15)


def unlane(y, k):
    """the data word w with lane(w, k) == y"""
    x = y ^ (y >> 15) ^ (y >> 30)
    return ((x * _MIX_INV) & M32) ^ (k * LANE_KEY & M32)


def fingerprint(data128):
    """the fingerprint k_intake_parse and k_api_parse compute of 128 AttestationData bytes"""
    assert len(data128) == 128
    h = 0
    for k in range(32):
        h ^= lane(_word(data128, k), k)
    return h


def with_fingerprint(d, target, fix_lane):
    """d with word fix_lane rewritten so that its fingerprint is target"""
    rest = fingerprint(d) ^ lane(_word(d, fix_lane), fix_lane)
    out = _set_word(d, fix_lane, unlane(target ^ rest, fix_lane))
    assert fingerprint(out) == target
    return out


def collide(d, change_lane, fix_lane, delta=1):
    """other data with d's fingerprint: word change_lane XOR delta, then word fix_lane fixed up"""
    assert change_lane != fix_lane and delta & M32
    out = with_fingerprint(_set_word(d, change_lane, _word(d, change_lane) ^ delta), fingerprint(d), fix_lane)
    assert out != d and fingerprint(out) == fingerprint(d)
    return out


def collision_set(d, variants, fix_lane):
    """[d] + every variant (data that differ from d outside word fix_lane) moved onto d's fingerprint through word fix_lane: distinct
    data, one fingerprint"""
    f = fingerprint(d)
    out = [bytes(d)] + [with_fingerprint(v, f, fix_lane) for v in variants]
    assert len(set(out)) == len(out) and {fingerprint(x) for x in out} == {f}
    return out


def source_lane_set(d, k, change_lane=14, fix_lane=15):
    """k distinct data with d's fingerprint that differ from d only in the source root (words change_lane and fix_lane): all valid
    wherever d is"""
    assert change_lane in FREE_LANES and fix_lane in FREE_LANES
    return collision_set(d, [_set_word(d, change_lane, _word(d, change_lane) ^ i) for i in range(1, k)], fix_lane)


def near_miss(root, byte, delta):
    """root with byte `byte` moved by delta (mod 256)"""
    r = bytearray(root)
    r[byte] = (r[byte] + delta) & 0xFF
    assert bytes(r) != bytes(root)
    return bytes(r)


def memcmp_less(a, b):
    return bytes(a) < bytes(b)


def le_word_less(a, b):
    """the order of a compare of little-endian 32-bit words, the wrong one for roots"""
    wa = [_word(a, k) for k in range(8)]
    wb = [_word(b, k) for k in range(8)]
    return wa < wb


PREFIX_BYTES = (0, 3, 4, 15, 16, 27, 28, 31)      # both ends of every 32-bit word and 16-byte half the device compares


def shared_prefix_groups(rng, positions=PREFIX_BYTES, per_group=3):
    """{p: roots}: per position p, per_group roots equal in every byte but p (byte p in ascending random order)"""
    groups = {}
    for p in positions:
        base = bytearray(rng.integers(0, 256, 32, dtype=np.uint8).tobytes())
        vals = sorted(rng.choice(np.arange(1, 255), per_group, replace=False).tolist())
        g = []
        for v in vals:
            base[p] = v
            g.append(bytes(base))
        assert all(sum(x != y for x, y in zip(g[0], r)) == 1 for r in g[1:])
        groups[p] = g
    return groups


def le_flip_pairs(rng, words=(0, 3, 4, 7)):
    """per word w, roots (a, b) equal but in word w, which holds 01 00 00 00 in a and 00 00 00 02 in b: memcmp puts b first, a compare
    of little-endian words puts a first"""
    pairs = []
    for w in words:
        base = bytearray(rng.integers(0, 255, 32, dtype=np.uint8).tobytes())
        base[4 * w:4 * w + 4] = b"\x01\x00\x00\x00"
        a = bytes(base)
        base[4 * w:4 * w + 4] = b"\x00\x00\x00\x02"
        b = bytes(base)
        assert memcmp_less(b, a) and le_word_less(a, b)
        pairs.append((a, b))
    return pairs


def edge_roots():
    """the smallest root and the largest that is not the oracle's outside marker"""
    return [bytes(32), b"\xff" * 31 + b"\xfe"]


def near_misses(root, tree_roots, deltas=(-1, 1)):
    """every one-byte +-1 neighbour of root that names no tree root and is not the outside marker"""
    known = set(tree_roots) | {OUTSIDE}
    out = []
    for byte in range(32):
        for dl in deltas:
            r = near_miss(root, byte, dl)
            if r not in known:
                out.append(r)
    return out
