"""tests/sync_keys.py against a direct evaluation of the sync intakes' home-slot formula, and the oracles' closed-form mode against their
default mode on small real-signature cases."""
import hashlib

import pytest

import scenarios
import sync_contributions_oracle as C
import sync_keys as K
import sync_messages_oracle as MO
from oracle import bls_sig as B
from oracle.bls12_381 import R


def _direct(root: bytes, tab: int) -> int:
    """the kernels' expression, step by step over 32-bit words"""
    h = root[0] | root[1] << 8 | root[2] << 16 | root[3] << 24
    h ^= (root[31] << 24) & 0xFFFFFFFF
    h = (h * 0x9E3779B9) % (1 << 32)
    return (h >> 7) & (tab - 1)


def test_table_size():
    assert [K.table_size(n) for n in (1, 2, 3, 64, 65, 4096)] == [2, 4, 8, 128, 256, 8192]


@pytest.mark.parametrize("tab", [2, 4, 8, 128, 256, 8192, 1 << 17, 1 << 25])
def test_root_at_lands_on_its_slot(tab):
    for slot in sorted({0, 1, tab // 2, tab - 2, tab - 1} & set(range(tab))):
        for tag in range(5):
            r = K.root_at(slot, tab, tag)
            assert len(r) == 32 and _direct(r, tab) == K.home_slot(r, tab) == slot
    assert len({K.root_at(tab - 1, tab, t) for t in range(50)}) == 50


def test_random_roots_agree_with_direct_formula():
    for i in range(2000):
        r = hashlib.sha256(i.to_bytes(4, "little")).digest()
        for tab in (2, 256, 8192, 1 << 20):
            assert K.home_slot(r, tab) == _direct(r, tab)


@pytest.mark.parametrize("k,tab", [(2, 4), (3, 8), (33, 128), (257, 8192), (300, 1 << 17)])
def test_colliding_roots(k, tab):
    rs = K.colliding(k, tab - 1, tab)
    assert len(set(rs)) == k and {_direct(r, tab) for r in rs} == {tab - 1}
    # each differs from the first at one byte; bytes 4-31 each take a turn when k allows
    diffs = [[i for i in range(32) if r[i] != rs[0][i]] for r in rs[1:]]
    assert all(len(d) == 1 and 4 <= d[0] <= 31 for d in diffs)
    assert {d[0] for d in diffs} == set(range(4, 4 + min(k - 1, 28)))


def test_byte_31_keeps_the_slot_up_to_2_17():
    r = bytearray(K.root_at(77, 1 << 17))
    for v in range(256):
        r[31] = v
        assert _direct(bytes(r), 1 << 17) == 77


# ---- closed-form mode of the oracles: the (secret key sum, signing root) pairs signed give the default mode's bytes

def _sign(keys, msgs):
    return [B.Sign(k, m) for k, m in zip(keys, msgs)]


def test_messages_closed_form_matches_default():
    sk = lambda v: scenarios.secret_key(v)      # noqa: E731
    pv = [3, 5, 5, 9, 11, 3, 13, 14]            # 2 subnets of 4; 5 twice in subnet 0, 3 on both subnets
    pks = {v: B.SkToPk(sk(v)) for v in set(pv)}
    dom, slot = bytes(range(32)), 4
    ra, rb = bytes([1] * 32), bytes([2] * 32)
    plan = [(3, 0, ra), (5, 0, ra), (9, 0, rb), (3, 1, rb), (13, 1, rb), (14, 1, ra)]
    wires = [MO.encode(slot, r, v, B.Sign(sk(v), MO.signing_root(r, dom))) for v, s, r in plan]
    subnets = [s for _, s, _ in plan]
    want = MO.validate(wires, subnets, pv, 16, lambda v: pks[v], slot, dom, count=2)
    cf = MO.validate(wires, subnets, pv, 16, lambda v: pks[v], slot, dom, count=2, secret_key=sk, closed_form=True)
    assert all(isinstance(p, tuple) for p in MO.closed_form_pairs(cf))
    MO.sign_closed_form(cf, _sign)
    assert cf.status == want.status == [0] * 6
    assert {k: c.signature for k, c in cf.contributions.items()} == {k: c.signature for k, c in want.contributions.items()}
    assert [a.sync_committee_signature for a in cf.aggregates] == [a.sync_committee_signature for a in want.aggregates]
    assert [a.sync_committee_bits for a in cf.aggregates] == [a.sync_committee_bits for a in want.aggregates]


def test_contributions_closed_form_matches_default():
    pv = list(range(16))                        # 4 subnets of 4
    dom, slot = bytes(range(96)), 6
    sg = C.Signer(pv, dom, slot)
    pks = {v: B.SkToPk(sg.sk(v)) for v in pv}
    ra, rb = bytes([1] * 32), bytes([2] * 32)
    on = lambda *ix: [i in ix for i in range(4)]      # noqa: E731
    wires = [sg.item(0, 0, ra, on(0, 1)), sg.item(5, 1, ra, on(1, 2, 3)), sg.item(6, 1, rb, on(0)), sg.item(10, 2, rb, on(2, 3))]
    want = C.validate(wires, pv, 16, lambda v: pks[v], slot, dom, target=16)
    cf = C.validate(wires, pv, 16, lambda v: pks[v], slot, dom, target=16, secret_key=sg.sk, closed_form=True)
    assert want.status == [0, 0, 0, 0] and len(want.roots) == 2
    MO.sign_closed_form(cf, _sign)
    assert cf.status == want.status and cf.best == want.best
    assert [a.sync_committee_signature for a in cf.aggregates] == [a.sync_committee_signature for a in want.aggregates]
    # a root whose keys cancel: the closed form gives the point at infinity, as bls.Aggregate does
    v, w = 0, 5
    sk = lambda x: (R - sg.sk(v)) if x == w else sg.sk(x)      # noqa: E731
    sg2 = C.Signer(pv, dom, slot, secret_key=sk)
    pk2 = {x: B.SkToPk(sk(x)) for x in pv}
    wires = [sg2.item(v, 0, ra, on(0)), sg2.item(w, 1, ra, on(1))]
    want = C.validate(wires, pv, 16, lambda x: pk2[x], slot, dom, target=16)
    cf = MO.sign_closed_form(C.validate(wires, pv, 16, lambda x: pk2[x], slot, dom, target=16, secret_key=sk, closed_form=True), _sign)
    assert want.status == [0, 0] and want.aggregates[0].sync_committee_signature == bytes([0xC0]) + bytes(95)
    assert cf.aggregates[0].sync_committee_signature == want.aggregates[0].sync_committee_signature
