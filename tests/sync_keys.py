"""beacon_block_roots that land on a chosen slot of the sync intakes' root tables (TEST INFRASTRUCTURE).

Both sync intakes (csrc/syncmsg.cuh k_scm_accept, csrc/synccontrib.cuh k_scc_parse) enter each accepted root in an insert-only table of
tab slots, tab the smallest power of two >= 2n, n the call's item count.  The home slot of a root r is

    h = ((le32(r[0:4]) ^ r[31] << 24) * 0x9e3779b9 mod 2^32) >> 7 & (tab - 1)

and a taken slot holding another root sends the probe on to h + 1 (mod tab), comparing all 32 bytes.  The multiplier is odd, so the hash
inverts: choose the product y with the wanted slot in bits 7 and up, then le32(r[0:4]) ^ r[31] << 24 = y * M^-1 mod 2^32.

Bytes 4-30 do not enter the hash, and byte 31 only moves bits 24-31 of the product (a change of r[31] changes the hashed word by a
multiple of 2^24, and so the product): for tables of up to 2^17 slots, roots that differ in any of bytes 4-31 share their home slot.
"""
M = 0x9E3779B9
M_INV = pow(M, -1, 1 << 32)


def table_size(n: int) -> int:
    """the root table's slot count for a call of n items"""
    tab = 1
    while tab < 2 * n:
        tab <<= 1
    return tab


def home_slot(root: bytes, tab: int) -> int:
    x = (int.from_bytes(root[0:4], "little") ^ root[31] << 24) & 0xFFFFFFFF
    return ((x * M) & 0xFFFFFFFF) >> 7 & (tab - 1)


def root_at(slot: int, tab: int, tag: int = 0) -> bytes:
    """a root whose home slot is `slot` in a table of tab slots; tag (any int) picks one of many such roots"""
    assert tab & (tab - 1) == 0 and 0 <= slot < tab <= 1 << 25
    hi = (tag * 0x2545F491) & 0xFFFFFFFF                        # the product's bits outside the slot
    y = (hi & ~((tab - 1) << 7) | slot << 7) & 0xFFFFFFFF
    x = (y * M_INV) & 0xFFFFFFFF
    fill = bytes((tag * 37 + 11 * i + 5) & 0xFF for i in range(27))
    last = (tag * 101 + 7) & 0xFF
    root = ((x ^ last << 24) & 0xFFFFFFFF).to_bytes(4, "little") + fill + bytes([last])
    assert home_slot(root, tab) == slot
    return root


def colliding(k: int, slot: int, tab: int, tag: int = 0):
    """k distinct roots on one home slot: the first from root_at, root j >= 1 differs from it at byte 4 + (j - 1) % 28 alone (bytes 4-31
    in turn, so the byte-31 near miss comes once in every 28) by the nonzero xor 1 + (j - 1) // 28"""
    assert tab <= 1 << 17 and k <= 28 * 255
    base = root_at(slot, tab, tag)
    out = [base]
    for j in range(1, k):
        r = bytearray(base)
        r[4 + (j - 1) % 28] ^= 1 + (j - 1) // 28
        out.append(bytes(r))
    assert len(set(out)) == k and all(home_slot(r, tab) == slot for r in out)
    return out
