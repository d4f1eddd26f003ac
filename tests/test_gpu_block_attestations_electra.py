"""Electra block attestations on the GPU (b2_block_attestations_electra / _dev, Engine.block_attestations_electra / _dev,
Spec.process_block_attestations_electra) against tests/block_attestations_electra_oracle.py byte for byte through both ABI forms and both
participation tables: every status 0-13, Deneb's inclusion window at 32-slot epochs, committee_bits patterns up to all 64, the Bitlist limit,
the split key sum's edges (segments around the chunk size, empty chunks, equal partial sums, partial sums that cancel, an invalid key in one
chunk), effective balances from below EFFECTIVE_BALANCE_INCREMENT to 2 048 ETH, block-atomic failure, the RLC verify mode, the device guards
and host refusals, the equivalence with b2_block_attestations for one-committee attestations, a 2^20-validator mainnet epoch of 32 blocks x 8
aggregates, and the Spec facade against the literal oracle block by block.  Signatures are made on the GPU by b2_sign with each aggregate's
summed secret key."""
import copy
import hashlib

import numpy as np
import pytest
import torch

import block_attestations_electra_oracle as E
import block_attestations_oracle as O
from oracle.bls12_381 import R
from pos_evolution_b200._lib import B2_EINVAL, B2Error
from pos_evolution_b200.engine import Engine
from test_gpu_block_attestations import DOMAINS, INC, PER_INC, KnownBLS, World, same

pytestmark = pytest.mark.gpu

CHUNK = 2048                   # BAE_CHUNK of csrc/blockatt_electra.cuh


def _h(b):
    return hashlib.sha256(b).digest()


class EWorld(World):
    """World with Electra attestations: M committee bits, Bitlist limit max_vpc * M; atts are signed in batches (sign())"""

    def __init__(self, eng, n_val, spe, e, cps_prev, cps_cur, sizes, M, max_vpc, seed):
        super().__init__(eng, n_val, spe, e, cps_prev, cps_cur, sizes, 1, seed)
        self.M, self.max_vpc, self.pending = M, max_vpc, []

    def eatt(self, slot, picks, bits=None, head=None, target=None, source=None, tepoch=None, index=0, corrupt=False, sign_with=None, sig=None):
        """a handle to the encoding of an attestation of the committees `picks` of slot, right unless told otherwise.  sign_with: the
        validators whose secret keys sign instead of the attesters; sig: the signature bytes.  Either makes the signature one the oracle's
        stand-in does not take as right."""
        Ep = slot // self.spe
        tepoch = Ep if tepoch is None else tepoch
        cps = self.cps_cur if Ep == self.e else self.cps_prev
        flat = [v for i in picks for v in (self.committee(slot, i) if i < cps else [0, 1, 2])]
        bits = [True] * len(flat) if bits is None else list(bits)
        if source is None:
            source = self.justified[40:80] if tepoch == self.e else self.justified[0:40]
        d = E.data128(slot, index, self.root(slot) if head is None else head, int.from_bytes(source[:8], "little"), source[8:], tepoch,
                      self.root(tepoch * self.spe) if 0 <= tepoch * self.spe - (self.e - 1) * self.spe < 2 * self.spe and target is None
                      else (target or bytes(32)))
        sel = sorted(set(v for v, b in zip(flat, bits) if b))
        msg = O.signing_root(d, DOMAINS[32:] if tepoch == self.e else DOMAINS[:32])
        sk = (sum(self.sks[v] for v in (sel if sign_with is None else sign_with)) + (1 if corrupt else 0)) % R or 1
        right = not corrupt and sign_with is None and sig is None
        self.pending.append((bits, d, sel, msg, sk, right, E.committee_bits_of(picks, self.M), sig))
        return len(self.pending) - 1

    def sign(self):
        """the encodings of every pending attestation, signed in one call"""
        P, self.pending = self.pending, []
        sigs = self.eng.sign([p[4] for p in P], np.arange(len(P), dtype=np.uint32), np.frombuffer(b"".join(p[3] for p in P), np.uint8).reshape(-1, 32))
        out = []
        for (bits, d, sel, msg, _, right, cb, given), sig in zip(P, sigs):
            if right:
                self.good[(tuple(sel), msg)] = bytes(sig)
            out.append(E.encode(bits, d, bytes(sig) if given is None else given, cb))
        return out

    def args(self, blocks, slots):
        a = super().args(blocks, slots)
        del a["bits_stride"]
        return dict(a, max_committees_per_slot=self.M, max_validators_per_committee=self.max_vpc)

    def host(self, a, t):
        self.eng.participation_load(0, t[0])
        self.eng.participation_load(1, t[1])
        r = self.eng.block_attestations_electra(**a)
        return r, self.eng.participation_read(0), self.eng.participation_read(1)

    def dev(self, a, t):
        eng = self.eng
        eng.participation_load(0, t[0])
        eng.participation_load(1, t[1])
        T = lambda x, dt: torch.from_numpy(np.ascontiguousarray(x, dtype=dt).copy()).cuda()      # noqa: E731
        r = eng.block_attestations_electra_dev(T(np.frombuffer(a["wire"], np.uint8), np.uint8), T(a["woff"], np.uint32), T(a["block_off"], np.uint32),
                                               T(a["block_slot"], np.uint64), T(a["members"], np.uint32), T(a["off"], np.uint32), a["cps_prev"],
                                               a["cps_cur"], T(a["chain_roots"], np.uint8), a["justified80"], a["domains64"], a["slots_per_epoch"],
                                               a["min_inclusion_delay"], a["max_committees_per_slot"], a["max_validators_per_committee"],
                                               E.row_max(a["off"], a["cps_prev"], a["cps_cur"], a["slots_per_epoch"]), INC, PER_INC)
        torch.cuda.synchronize()
        o = [x.cpu().numpy() for x in r]
        return (o[0], o[1], o[2], o[3], o[4], o[5], int(o[6][0])), eng.participation_read(0), eng.participation_read(1)

    def oracle(self, a, t):
        return E.run(a["wire"], a["woff"], a["block_off"], a["block_slot"], self.members, self.off, self.cps_prev, self.cps_cur, self.roots,
                     self.justified, DOMAINS, self.spe, 1, self.M, self.max_vpc, self.eff, INC, PER_INC, t[0].tolist(), t[1].tolist(), self.verify)

    def both(self, handles, slots, seed=0):
        """both forms against the oracle on blocks given as lists of handles (or raw encodings)"""
        enc = self.sign()
        blocks = [[enc[h] if isinstance(h, int) else h for h in blk] for blk in handles]
        a, t = self.args(blocks, slots), self.tables(seed)
        o = self.oracle(a, t)
        same(self.host(a, t), o)
        same(self.dev(a, t), o)
        return o


@pytest.fixture(scope="module")
def W():
    # e = 3 on 4-slot epochs (slots 12-15), 2 committees per slot in e - 1 and 3 in e, M = 4, ragged committees of 3-24, limit 4 * 24
    return EWorld(Engine(0), 400, 4, 3, 2, 3, list(range(3, 25)), 4, 24, 1)


def test_every_status_through_both_forms(W):
    s = 14
    F = E.fixed(4)
    good = W.eatt(13, [0, 1])
    bad = [W.eatt(12, [0, 2]), W.eatt(13, [1]), W.eatt(13, [2]), W.eatt(5, [0], tepoch=1), W.eatt(9, [0], tepoch=3), W.eatt(14, [0]),
           W.eatt(13, [0], index=1), W.eatt(13, [0, 3]), W.eatt(13, [0, 1], bits=[True] * len(W.committee(13, 0)) + [False] * len(W.committee(13, 1))),
           W.eatt(13, [0, 1], bits=[True] * (len(W.committee(13, 0)) + len(W.committee(13, 1)) - 1)), W.eatt(13, [1], source=W.justified[:40]),
           W.eatt(13, []), W.eatt(12, [2], corrupt=True)]
    enc = W.sign()
    g = enc[good]
    raw = [g[:F - 1], bytes([F + 1]) + g[1:], g[:F - 1] + bytes([g[F - 1] | 0x20]) + g[F:], g[:F], g[:-1] + bytes(1),
           g[:F] + E.bitlist([True] * (4 * 24 + 1))]
    blk1 = [enc[bad[1]]] + raw[:1] + raw[3:4] + raw[5:6] + [enc[h] for h in bad[3:]]
    blocks = [[enc[bad[0]]], blk1, [enc[bad[2]]]]
    # block 0: committees (12, 0) and (12, 2) valid; block 1: a valid one then statuses 1-13; block 2 valid but after the invalid block
    a, t = W.args(blocks, [13, s, 15]), W.tables(0)
    o = W.oracle(a, t)
    same(W.host(a, t), o)
    same(W.dev(a, t), o)
    assert o["status"].tolist() == [0, 0] + list(range(1, 14)) + [0] and o["n_applied"] == 1 and o["block_status"].tolist() == [0, 1, 2]
    assert o["block_first"].tolist() == [0xFFFFFFFF, 1, 0xFFFFFFFF]
    # the other malformed containers: a wrong offset, a padding bit of committee_bits, no delimiter
    for r, st in ((raw[1], 1), (raw[2], 1), (raw[4], 2)):
        a = W.args([[r]], [14])
        o = W.oracle(a, t)
        same(W.host(a, t), o)
        same(W.dev(a, t), o)
        assert o["status"].tolist() == [st]


def test_block_atomic_failure_and_reinclusion(W):
    """an invalid block in the middle; a repeated aggregate and a sub-aggregate earn nothing"""
    half = [j % 2 == 0 for j in range(len(W.committee(12, 0)) + len(W.committee(12, 1)))]
    o = W.both([[W.eatt(12, [0, 1]), W.eatt(11, [0, 1])], [W.eatt(12, [0, 1]), W.eatt(12, [0, 1], bits=half), W.eatt(13, [1, 2])],
                [W.eatt(14, [0]), W.eatt(13, [0], corrupt=True)]], [13, 14, 15], seed=3)
    assert o["n_applied"] == 2 and o["status"].tolist() == [0, 0, 0, 0, 0, 0, 13] and o["numerator"].tolist()[2:4] == [0, 0]
    assert o["block_status"].tolist() == [0, 0, 1] and o["block_reward"][2] == 0


def test_rlc_mode_gives_identical_outputs(W):
    hs = [[W.eatt(13, [0, 2]), W.eatt(12, [1])], [W.eatt(13, [1]), W.eatt(12, [0, 1], corrupt=True), W.eatt(10, [0, 1])]]
    enc = W.sign()
    a, t = W.args([[enc[h] for h in b] for b in hs], [14, 15]), W.tables(5)
    ref = W.host(a, t)
    W.eng.set_verify_mode(True, bytes(range(32)))
    try:
        got = W.host(a, t)
        dev = W.dev(a, t)
    finally:
        W.eng.set_verify_mode(False)
    o = W.oracle(a, t)
    same(ref, o)
    same(got, o)
    same(dev, o)


@pytest.fixture(scope="module")
def W32():
    # e = 2 on 32-slot epochs (slots 64-95; e - 1 = 32-63), 64 committees per slot of 1-3 members, M = 64
    return EWorld(Engine(0), 12800, 32, 2, 64, 64, [1, 2, 3], 64, 3, 2)


def test_deneb_inclusion_delays(W32):
    """delays 1, 5, 6, 32, 33 and 63 from slot 95: source up to 5, target throughout, head only at 1"""
    W = W32
    hs = [W.eatt(95 - d, [0, 5]) for d in (1, 5, 6, 32, 33, 63)] + [W.eatt(90, [1], head=_h(b"h")), W.eatt(40, [2], target=_h(b"t"))]
    o = W.both([hs], [95])
    assert o["status"].tolist() == [0] * 8 and o["flag_mask"].tolist() == [7, 3, 2, 2, 2, 2, 3, 0]


def test_committee_bit_patterns(W32):
    """single, first, last (63), all 64 and alternating committee_bits; the previous epoch's too"""
    W = W32
    pats = [[17], [0], [63], list(range(64)), list(range(0, 64, 2)), list(range(1, 64, 2))]
    hs = [W.eatt(80, p) for p in pats] + [W.eatt(50, p) for p in pats]
    o = W.both([hs[:6], hs[6:]], [81, 82], seed=7)
    assert o["status"].tolist() == [0] * 12 and o["n_applied"] == 2


def test_bitlist_limit():
    """committees of exactly max_validators_per_committee: a two-committee aggregate at the limit is valid, one bit more is status 3"""
    W = EWorld(Engine(0), 200, 4, 3, 2, 2, [5], 2, 5, 3)
    h = W.eatt(13, [0, 1])
    enc = W.sign()
    F = E.fixed(2)
    over = enc[h][:F] + E.bitlist([True] * 11)
    a, t = W.args([[enc[h], over]], [14]), W.tables(1)
    o = W.oracle(a, t)
    same(W.host(a, t), o)
    same(W.dev(a, t), o)
    assert o["status"].tolist() == [0, 3]


@pytest.fixture(scope="module")
def WS():
    # e = 2 on 2-slot epochs (slots 4-5; e - 1 = 2-3), the committees of every slot of CHUNK - 1, CHUNK and CHUNK + 1 members: rows of
    # 3 CHUNK members
    W = EWorld(Engine(0), 12 * CHUNK + 16, 2, 2, 3, 3, [CHUNK], 3, 4096, 4)
    W.off = np.concatenate([[0], np.cumsum([CHUNK - 1, CHUNK, CHUNK + 1] * 4)]).astype(np.uint32)
    W.members = np.random.default_rng(4).permutation(W.n_val)[:int(W.off[-1])].astype(np.uint32)
    return W


def test_split_sum_segment_edges(WS):
    """segments of CHUNK - 1, CHUNK and CHUNK + 1 members alone and together, chunks without a set bit, bits on each side of the chunk
    edges, a row whose only set bit is its first and one whose only set bit is its last"""
    W = WS
    sizes = [len(W.committee(4, i)) for i in range(3)]
    assert sizes == [CHUNK - 1, CHUNK, CHUNK + 1]
    total = sum(sizes)
    edge = [j in (0, CHUNK - 1, CHUNK, 2 * CHUNK - 1, 2 * CHUNK) for j in range(total)]
    prev = [len(W.committee(3, i)) for i in range(3)]
    hs = [W.eatt(4, [0]), W.eatt(4, [1]), W.eatt(4, [2]), W.eatt(4, [0, 1, 2]), W.eatt(4, [0, 1, 2], bits=edge),
          W.eatt(3, [0, 2], bits=[True] + [False] * (prev[0] + prev[2] - 2) + [True]),
          W.eatt(3, [1], bits=[j == 0 for j in range(prev[1])]), W.eatt(2, [2], bits=[j == sizes[2] - 1 for j in range(len(W.committee(2, 2)))])]
    o = W.both([hs], [5], seed=1)
    assert o["status"].tolist() == [0] * 8


def test_split_sum_equal_cancelling_and_invalid_partials(WS):
    """aggregates of committees 0 and 2 (rows of 2 CHUNK members, two chunks): a key duplicated in both chunks (the combine doubles), keys sk
    and r - sk in the two chunks (the sum is infinity: the aggregate fails as b2_fast_aggregate_verify fails such a set), and an invalid
    registry key in one chunk (13).  The last two carry the signature the pairing accepts when their PK_INFINITY or PK_INVALID_KEY bit is
    lost: the G2 identity (e(inf, H(m)) = e(g1, inf)), and the secret-key sum of the other attesters (the gather skips the invalid key's
    zero record), so only the combine's status bits make them 13."""
    W = WS
    com = W.committee(4, 0) + W.committee(4, 2)
    i0, i1, i2, i3, i4 = com[5], com[CHUNK + 576], com[10], com[CHUNK + 476], com[CHUNK + 76]
    sks = list(W.sks)
    sks[i1] = sks[i0]                          # equal partial sums
    sks[i3] = R - sks[i2]                      # partial sums that cancel
    pk = W.eng.sk_to_pk(sks)
    pk[i4] = np.frombuffer(bytes([0xA0]) + bytes(47), np.uint8)      # x = 0: not in G1, KeyValidate fails
    identity = bytes([0xC0]) + bytes(95)
    try:
        W.sks = sks
        assert W.eng.registry_load(pk, W.eff)[i4] == 0
        dup = W.eatt(4, [0, 2], bits=[j in (5, CHUNK + 576) for j in range(len(com))])
        both = W.eatt(4, [0, 2], bits=[j in (5, CHUNK + 576, 9) for j in range(len(com))])
        # FastAggregateVerify is False for these (an infinity aggregate key, a key that fails KeyValidate)
        cancel = W.eatt(4, [0, 2], bits=[j in (10, CHUNK + 476) for j in range(len(com))], sig=identity)
        invalid = W.eatt(4, [0, 2], bits=[j in (1, CHUNK + 76) for j in range(len(com))], sign_with=[com[1]])
        o = W.both([[dup, both, cancel, invalid]], [5], seed=2)
        assert o["status"].tolist() == [0, 0, 13, 13]
        msg = np.frombuffer(_h(b"cancel"), np.uint8).reshape(1, 32)
        sig = np.frombuffer(identity, np.uint8).reshape(1, 96)
        assert W.eng.fast_aggregate_verify([i2, i3], [0, 2], np.array([[3]], np.uint8), msg, sig).tolist() == [0]
    finally:
        W.sks = [i + 1 for i in range(W.n_val)]
        W.eng.registry_load(W.eng.sk_to_pk(W.sks), W.eff)


def test_effective_balances_from_below_an_increment_to_2048_eth(WS):
    W = WS
    rng = np.random.default_rng(3)
    eff = W.eff.copy()
    W.eff = (rng.choice([2048 * 10**9, 1024 * 10**9 + 7, 5 * 10**8, 10**9 - 1, 32 * 10**9, 0], W.n_val)).astype(np.uint64)
    try:
        W.eng.registry_load(W.eng.sk_to_pk(W.sks), W.eff)
        o = W.both([[W.eatt(3, [0, 1, 2]), W.eatt(2, [1])], [W.eatt(4, [0], bits=[j % 3 == 0 for j in range(len(W.committee(4, 0)))])]], [4, 5], seed=4)
        assert o["status"].tolist() == [0, 0, 0] and (o["block_reward"] > 0).all()
    finally:
        W.eff = eff
        W.eng.registry_load(W.eng.sk_to_pk(W.sks), W.eff)


def test_device_guards(W):
    hs = [[W.eatt(13, [0, 1])], [W.eatt(13, [2]), W.eatt(12, [0])]]
    enc = W.sign()
    a, t = W.args([[enc[h] for h in b] for b in hs], [14, 15]), W.tables(2)

    def call(mutate):
        x = dict(a)
        mutate(x)
        W.eng.guard_flags()
        got = W.dev(x, t)
        return got, W.eng.guard_flags()

    def woff(x):
        x["woff"] = x["woff"].copy()
        x["woff"][2] = x["woff"][1] - 1
    got, g = call(woff)
    assert got[0][0][1] == 1 and got[0][3].tolist() == [0, 1] and g & 2

    def off(x):
        x["off"] = x["off"].copy()
        x["off"][W.cps_prev * W.spe + 1 * W.cps_cur + 1] = len(x["members"]) + 5      # committee (13, 0) ends past the members
    got, g = call(off)
    assert got[0][0][0] == 10 and got[0][6] == 0 and g & 2

    # a member index past the registry, in an aggregate signed by the other attesters' keys: it verifies unless PK_BAD_INDEX holds it (13)
    com = W.committee(13, 2)
    hm = W.eatt(13, [2], sign_with=com[1:])
    enc_m = W.sign()
    a = W.args([[enc[hs[0][0]]], [enc_m[hm]]], [14, 15])

    def member(x):
        x["members"] = x["members"].copy()
        x["members"][x["off"][W.cps_prev * W.spe + 1 * W.cps_cur + 2]] = W.n_val + 7      # the first member of committee (13, 2)
    got, g = call(member)
    assert got[0][0].tolist() == [0, 13] and got[0][6] == 1 and g & 1


def test_host_refusals_change_nothing(W):
    hs = [[W.eatt(13, [0, 1])], [W.eatt(13, [2])]]
    enc = W.sign()
    a, t = W.args([[enc[h] for h in b] for b in hs], [14, 15]), W.tables(4)
    W.eng.participation_load(0, t[0])
    W.eng.participation_load(1, t[1])
    bad = [dict(a, max_committees_per_slot=0), dict(a, max_committees_per_slot=65), dict(a, max_validators_per_committee=0),
           dict(a, max_validators_per_committee=1 << 30), dict(a, block_slot=np.array([15, 14], np.uint64)), dict(a, cps_prev=3)]
    x = dict(a)
    x["woff"] = x["woff"].copy()
    x["woff"][-1] = len(x["wire"]) + 1
    bad.append(x)
    x = dict(a)
    x["off"] = x["off"].copy()
    x["off"][1], x["off"][2] = x["off"][2], x["off"][1]
    bad.append(x)
    for x in bad:
        with pytest.raises(B2Error) as err:
            W.eng.block_attestations_electra(**x)
        assert err.value.code == B2_EINVAL
    assert W.eng.participation_read(0).tolist() == t[0].tolist() and W.eng.participation_read(1).tolist() == t[1].tolist()
    eng = Engine(0)
    with pytest.raises(B2Error) as err:
        eng.block_attestations_electra(**a)
    assert err.value.code == B2_EINVAL


def test_single_committee_matches_block_attestations(W):
    """one-committee Electra attestations within the Altair window: the outputs and tables of b2_block_attestations on their phase 0 forms"""
    plan = [[(12, 0), (12, 2), (11, 1), (10, 0)], [(13, 1), (12, 0), (11, 1)], [(14, 2), (12, 0)]]
    row = lambda s, c: [(j + c) % 3 != 1 for j in range(len(W.committee(s, c)))]      # noqa: E731
    hs = [[W.eatt(s, [c], bits=row(s, c)) for s, c in blk] for blk in plan]
    enc = W.sign()
    eblocks = [[enc[h] for h in blk] for blk in hs]
    pblocks = [[W.att(s, c, bits=row(s, c)) for s, c in blk] for blk in plan]      # data.index = c, signed over that data
    slots = [13, 14, 15]
    a, t = W.args(eblocks, slots), W.tables(6)
    W.eng.participation_load(0, t[0])
    W.eng.participation_load(1, t[1])
    ea = W.host(a, t)
    pa = World.args(W, pblocks, slots)
    pa["bits_stride"] = 4
    pr = World.host(W, pa, t)
    assert ea[0].status.tolist() == [0] * 9 and ea[0].n_applied == 3
    for x, y in zip(ea[0], pr[0]):
        assert np.asarray(x).tolist() == np.asarray(y).tolist()
    assert ea[1].tolist() == pr[1].tolist() and ea[2].tolist() == pr[2].tolist()


def test_full_size_electra_epoch_against_the_oracle():
    """2^20 validators on the mainnet preset (64 committees of 512 a slot), 32 blocks of 8 aggregates: block k at slot start(e) + k
    carries 8 aggregates of the slots before it, each naming about 95 % of that slot's 64 committees with about 95 % of their bits; the
    call's arguments from Spec.block_attestations_electra_inputs, both forms and both tables against the oracle"""
    from pos_evolution_b200 import spec as PS
    SPE, EP = 32, 3
    START = EP * SPE
    n, part = 1 << 20, 0.95
    eng = Engine(0)
    pspec = PS.Spec(PS.MAINNET, engine=eng)
    p = PS.MAINNET
    H = p.SLOTS_PER_HISTORICAL_ROOT
    sk0 = int.from_bytes(_h(b"electra/sk0"), "big") % (R >> 1) or 1
    delta = int.from_bytes(_h(b"electra/skd"), "big") >> 64
    sk8 = np.frombuffer(b"".join((sk0 + i * delta).to_bytes(32, "little") for i in range(n)), np.uint32).reshape(n, 8)
    pk = eng.sk_to_pk(sk8)
    state = PS.BeaconState(slot=START, fork=PS.Fork(), genesis_validators_root=bytes(32),
                           validators=[PS.Validator(pk[i].tobytes(), 32 * 10**9) for i in range(n)], balances=[32 * 10**9] * n,
                           randao_mixes=[_h(b"mix" + i.to_bytes(8, "little")) for i in range(p.EPOCHS_PER_HISTORICAL_VECTOR)],
                           block_roots=[_h(b"root" + s.to_bytes(8, "little")) for s in range(H)],
                           previous_epoch_participation=[0] * n, current_epoch_participation=[0] * n,
                           previous_justified_checkpoint=PS.Checkpoint(EP - 2, _h(b"j-prev")),
                           current_justified_checkpoint=PS.Checkpoint(EP - 1, _h(b"j-cur")))
    rng = np.random.default_rng(8)
    committees = {ep: pspec.epoch_committees(state, ep) for ep in (EP - 1, EP)}
    blocks, sks, msgs, sels = [], [], [], []
    for k in range(SPE):
        s = START + k
        atts = []
        for j in range(8):
            slot = s - 1 - j
            ep = slot // SPE
            members, off, cps = committees[ep]
            picks = [i for i in range(cps) if rng.random() < part] or [0]
            bits, sel = [], []
            for i in picks:
                c = (slot - ep * SPE) * cps + i
                com = members[off[c]:off[c + 1]]
                row = rng.random(len(com)) < part
                bits += row.tolist()
                sel += com[row].tolist()
            src = state.current_justified_checkpoint if ep == EP else state.previous_justified_checkpoint
            data = PS.AttestationData(slot, 0, bytes(state.block_roots[slot % H]), src, PS.Checkpoint(ep, bytes(state.block_roots[(ep * SPE) % H])))
            sks.append((sum(sel) * delta + len(sel) * sk0) % R)
            msgs.append(pspec.compute_signing_root(data, pspec.get_domain(state, PS.DOMAIN_BEACON_ATTESTER, ep)))
            sels.append(tuple(sorted(sel)))
            atts.append(PS.ElectraAttestation(bits, data, None, [i in set(picks) for i in range(64)]))
        blocks.append(PS.BlockAttestations(s, 0, bytes(state.block_roots[s % H]), atts))
    sigs = eng.sign(np.frombuffer(b"".join(v.to_bytes(32, "little") for v in sks), np.uint32).reshape(-1, 8), np.arange(len(sks), dtype=np.uint32),
                    np.frombuffer(b"".join(msgs), np.uint8).reshape(-1, 32))
    good = {}
    for j, a in enumerate(a for b in blocks for a in b.attestations):
        a.signature = sigs[j].tobytes()
        good[(sels[j], msgs[j])] = a.signature
    a = pspec.block_attestations_electra_inputs(state, blocks)
    assert a["max_committees_per_slot"] == 64 and len(a["woff"]) == 257
    pspec.sync_registry(state)
    t = [(rng.integers(0, 8, n) * (rng.random(n) < 0.3)).astype(np.uint8) for _ in range(2)]
    o = E.run(a["wire"], a["woff"], a["block_off"], a["block_slot"], a["members"], a["off"], a["cps_prev"], a["cps_cur"],
              a["chain_roots"].reshape(-1, 32), a["justified80"], a["domains64"], SPE, 1, 64, a["max_validators_per_committee"],
              np.full(n, 32 * 10**9, np.uint64), a["increment"], a["base_reward_per_increment"], t[0].tolist(), t[1].tolist(),
              lambda idx, root, sig: good.get((tuple(idx), bytes(root))) == bytes(sig))
    assert o["n_applied"] == SPE and not o["status"].any() and (o["block_reward"] > 0).all()
    eng.participation_load(0, t[0])
    eng.participation_load(1, t[1])
    res = eng.block_attestations_electra(**a)
    same((tuple(res), eng.participation_read(0), eng.participation_read(1)), o)
    T = lambda x, dt: torch.from_numpy(np.ascontiguousarray(x, dtype=dt).copy()).cuda()      # noqa: E731
    eng.participation_load(0, t[0])
    eng.participation_load(1, t[1])
    r = eng.block_attestations_electra_dev(T(np.frombuffer(a["wire"], np.uint8), np.uint8), T(a["woff"], np.uint32), T(a["block_off"], np.uint32),
                                           T(a["block_slot"], np.uint64), T(a["members"], np.uint32), T(a["off"], np.uint32), a["cps_prev"],
                                           a["cps_cur"], T(a["chain_roots"], np.uint8), a["justified80"], a["domains64"], SPE, 1, 64,
                                           a["max_validators_per_committee"], E.row_max(a["off"], a["cps_prev"], a["cps_cur"], SPE),
                                           a["increment"], a["base_reward_per_increment"])
    torch.cuda.synchronize()
    r = [x.cpu().numpy() for x in r]
    same(((r[0], r[1], r[2], r[3], r[4], r[5], int(r[6][0])), eng.participation_read(0), eng.participation_read(1)), o)
    eng.close()


def test_spec_run_matches_the_literal_oracle_block_by_block():
    """Spec.process_block_attestations_electra on the minimal preset over four blocks with skipped slots, each with its own proposer,
    against the pyspec-shaped Electra process_attestation of tests/test_oracle_block_attestations_electra.py block by block: every block
    valid, then a run whose third block holds a bad signature"""
    import scenarios
    import test_golden as TG
    import test_oracle_block_attestations_electra as TO
    from oracle import spec as OS
    from pos_evolution_b200 import spec as PS
    eng = Engine(0)
    pspec = PS.Spec(PS.MINIMAL, engine=eng)
    ospec = OS.Spec(OS.MINIMAL, bls_module=KnownBLS)
    spe, H = OS.MINIMAL.SLOTS_PER_EPOCH, OS.MINIMAL.SLOTS_PER_HISTORICAL_ROOT
    _, base = scenarios.minimal_state(64, slot=17, pks=TG.PKS)
    base.previous_justified_checkpoint = OS.Checkpoint(1, _h(b"j1"))
    base.current_justified_checkpoint = OS.Checkpoint(2, _h(b"j2"))
    slots = [17, 19, 20, 23]
    roots = [_h(b"erun" + bytes([s])) for s in slots]

    def root(s):
        return bytes(base.block_roots[s % H]) if s < slots[0] else [r for r, b in zip(roots, slots) if b <= s][-1]

    def att(s, picks, bits=None, corrupt=False):
        E_ = s // spe
        flat = [v for i in picks for v in ospec.get_beacon_committee(base, s, i)]
        bits = [True] * len(flat) if bits is None else bits
        src = base.current_justified_checkpoint if E_ == 2 else base.previous_justified_checkpoint
        data = OS.AttestationData(s, 0, root(s), src, OS.Checkpoint(E_, root(E_ * spe)))
        msg = ospec.compute_signing_root(data, ospec.get_domain(base, OS.DOMAIN_BEACON_ATTESTER, E_))
        sel = sorted(set(v for v, b in zip(flat, bits) if b))
        sk = (sum(scenarios.secret_key(v) for v in sel) + (1 if corrupt else 0)) % R
        sig = bytes(eng.sign([sk], [0], np.frombuffer(msg, np.uint8).reshape(1, 32))[0])
        if not corrupt:
            KnownBLS.good[(tuple(bytes(TG.PKS[v]) for v in sel), msg)] = sig
        return TO.Att(bits, data, sig, E.committee_bits_of(picks, 4))

    def product(a):
        d = a.data
        return PS.ElectraAttestation(list(a.aggregation_bits), PS.AttestationData(d.slot, d.index, d.beacon_block_root,
                                                                                  PS.Checkpoint(d.source.epoch, d.source.root),
                                                                                  PS.Checkpoint(d.target.epoch, d.target.root)), a.signature,
                                     list(a.committee_bits))

    def check(blocks):
        st, failed = copy.deepcopy(base), None
        for k, s in enumerate(slots):
            if k:
                for t in range(slots[k - 1], s):
                    st.block_roots[t % H] = roots[k - 1]
            st.slot = s
            before = copy.deepcopy(st)
            try:
                for a in blocks[k]:
                    TO.electra_process_attestation(ospec, st, a)
            except AssertionError:
                st, failed = before, k
                break
        proposers = []
        for s in slots:
            at = copy.copy(base)
            at.slot = s
            proposers.append(ospec.get_beacon_proposer_index(at))
        ps = TG._pstate(PS, base)
        n, statuses = pspec.process_block_attestations_electra(ps, [PS.BlockAttestations(s, p, r, [product(a) for a in blk])
                                                                    for s, p, r, blk in zip(slots, proposers, roots, blocks)])
        assert n == (len(slots) if failed is None else failed)
        assert ps.balances == st.balances
        assert ps.current_epoch_participation == st.current_epoch_participation
        assert ps.previous_epoch_participation == st.previous_epoch_participation
        return n, statuses

    run = [[att(16, [0, 1]), att(13, [0])],
           [att(18, [1]), att(17, [0, 1]), att(8, [0, 1])],
           [att(19, [0]), att(18, [0, 1], bits=[True, False] * 4), att(18, [0])],
           [att(22, [0, 1]), att(20, [1]), att(9, [1])]]
    n, statuses = check(run)
    assert n == 4 and all(not s.any() for s in statuses)
    run[2] = [att(19, [0]), att(18, [1], corrupt=True), att(18, [0])]
    n, statuses = check(run)
    assert n == 2 and statuses[2].tolist() == [0, 13, 0]
