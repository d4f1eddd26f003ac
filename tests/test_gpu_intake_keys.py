"""Both device intakes on adversarial keys (tests/intake_keys.py): AttestationData that share the 32-bit fingerprint the kernels compare
before the 128 data bytes, and block roots that differ from a tree root, or from each other, in one byte.

  A  the attestation intake (b2_attestation_intake / _dev): committees of 64, 512 and 2 048 members each holding K = 2, 3, 33 or 257
     distinct data on one fingerprint, interleaved, duplicated across colliding data, a failing datum ahead of a passing one
  B  the aggregate intake (b2_aggregate_and_proof_intake / _dev): a colliding datum is not shadowed by an accepted item of the other
     (check 10) while a byte-equal one is; fingerprint clusters on the last slot of the data table, so that probes wrap to slot 0, with
     byte-equal duplicates behind them; one batch on a single fingerprint; tables of 2 to 8 192 slots
  C  roots: a tree of roots sharing 31 bytes (differing at byte 0, 3, 4, 15, 16, 27, 28 or 31), pairs whose order flips under a compare
     of little-endian words, 00..00 and ff..fe; loaded, appended by b2_tree_add and pruned, and a one-block tree: every root is found with
     its block id, every one-byte neighbour is not, and the tied fan of each group has the head of oracle.fast and of a fresh load
  D  one committee flooded: 8 192 attestations in one 2 048-member committee, 2 048 aggregates in one committee (wall times printed)
  E  a committee split between two colliding data, both valid, through EpochProcessor.intake_dev and process_epoch_dev

Every output of both ABI forms is compared byte for byte with tests/intake_oracle.py or tests/aggregate_intake_oracle.py; the device
forms write into views inside sentinel-filled buffers, and nothing outside a view may change."""
import time
import types

import numpy as np
import pytest
import torch

import aggregate_intake_oracle as AO
import intake_keys as K
import intake_oracle as IO
import scenarios
import test_gpu_aggregate_intake as G
import test_gpu_tree_update as TU
from intake_oracle import data128 as make_data
from oracle import fast
from oracle.spec import Spec
from test_gpu_intake_shapes import DEV, DOMAIN, EPOCH, NONE, _check_dev, _check_host, _Padded, _wire

pytestmark = pytest.mark.gpu

FP = 0xC0111DE5                       # the fingerprint every collision set of A shares
NO_SIG = (False, False, False)        # the verdicts of an unsigned item (it fails before check 14, or fails check 14)


@pytest.fixture(scope="module")
def eng():
    from pos_evolution_b200.engine import Engine
    e = Engine(0)
    yield e
    e.close()


@pytest.fixture(scope="module")
def agg():
    """test_gpu_aggregate_intake's world: its registry and committees (each test loads the tree it needs)"""
    from pos_evolution_b200.engine import Engine
    e = Engine(0)
    sks = list(range(1, G.N_VAL + 1))
    e.registry_load(e.sk_to_pk(sks), np.full(G.N_VAL, 32 * 10**9, np.uint64))
    rng = np.random.default_rng(11)
    members = rng.permutation(G.N_VAL)[:sum(G.SIZES)].astype(np.uint32)
    off = np.concatenate([[0], np.cumsum(G.SIZES)]).astype(np.uint32)
    yield e, sks, members, off
    e.close()


def _numpy_oracle(tree, wires, off, spe, cps, stride):
    rec = np.frombuffer(b"".join(wires), np.uint8).reshape(len(wires), -1)
    return IO.intake_numpy(rec, np.asarray(off, np.int64), EPOCH, (EPOCH + 1) * spe, DOMAIN, cps, spe, stride, *tree)


def _intake_both(eng, wires, off, spe, cps, stride, want):
    """both forms of the attestation intake on the loaded tree against the oracle"""
    mv = int(want.vote_off[-1])
    _check_dev(eng, wires, off, spe, cps, stride, mv, want)
    _check_host(eng, wires, off, spe, cps, stride, mv, want)


def _att(size, p, d, rng):
    return IO.encode([j == p for j in range(size)], d, rng.integers(0, 256, 96, dtype=np.uint8).tobytes())


def _good_heads(tree, s, start):
    parent, slot, _ = tree
    return [b for b in range(len(parent)) if int(slot[b]) <= s and IO.ancestor(parent, slot, b, start) is not None] or [0]


# ------------------------------------------------------------------------------------------ A: the attestation intake
def _collision_epoch(seed, size, k, spe=2, cps=2):
    """(tree, wires, off, per-committee collision sets): every committee of `size` members holds k distinct data on fingerprint FP.
    The wires: per committee, three attestations of a failing datum first (each then loses its position to a later passing one); the
    members' attestations in random order; then second attestations of a sixteenth of the positions (at least four), with the first
    datum of the set or any other."""
    rng = np.random.default_rng(seed)
    tree = IO.random_tree(rng, 40, EPOCH * spe - 5)
    parent, slot, roots = tree
    _, ids = IO.block_store(*tree)
    rl = [bytes(r) for r in roots]
    start = EPOCH * spe
    front, body, late, sets = [], [], [], []
    for c in range(spe * cps):
        s = start + c // cps
        ok = _good_heads(tree, s, start)
        h = ok[int(rng.integers(len(ok)))]
        x = K.with_fingerprint(make_data(s, c % cps, rl[h], EPOCH - 1, rl[0], EPOCH, rl[IO.ancestor(parent, slot, h, start)]), FP, 20)
        variants = []
        for i in range(1, k):
            v = K._set_word(x, 14, K._word(x, 14) ^ i)                 # every variant differs in the source root ...
            if i % 4 == 2 and len(ok) > 1:                              # ... and may name another tree block as its head (words 4..11)
                v = v[:16] + rl[ok[(ok.index(h) + i) % len(ok)]] + v[48:]
            elif i % 4 == 3:                                            # ... or an unknown target (word 31): check 10
                v = K._set_word(v, 31, K._word(v, 31) ^ (i << 8 | 1))
            elif i % 4 == 0:                                            # ... or a known block as target, mostly not the ancestor: 12
                v = v[:96] + rl[int(rng.integers(len(rl)))]
            variants.append(v)
        data = K.collision_set(x, variants, 15)
        sets.append(data)
        fails = [d for d in data if IO._tree_check(d, ids, parent, slot, rl, start)[0] != 0]
        present = np.nonzero(rng.random(size) >= 0.1)[0]
        group = rng.permutation(np.arange(len(present)) % k)
        body += [(c, p, data[g]) for p, g in zip(present.tolist(), group.tolist())]
        if fails:
            front += [(c, p, fails[0]) for p in present[:3].tolist()]
        dup = rng.choice(present, max(4, len(present) // 16), replace=False).tolist()
        late += [(c, p, data[0] if j % 2 else data[int(rng.integers(k))]) for j, p in enumerate(dup)]
    order = rng.permutation(len(body))
    items = front + [body[i] for i in order] + late
    return tree, [_att(size, p, d, rng) for _, p, d in items], IO.ragged_layout([size] * spe * cps), sets


@pytest.mark.parametrize("k", [2, 3, 33, 257])
@pytest.mark.parametrize("size", [64, 512, 2048])
def test_intake_collision_sets(eng, size, k):
    stride = size // 8
    tree, wires, off, sets = _collision_epoch(100 * k + size, size, k)
    assert {K.fingerprint(bytes(w[4:132])) for w in wires} == {FP}
    want = _numpy_oracle(tree, wires, off, 2, 2, stride)
    st = set(want.status.tolist())
    assert 0 in st and 13 in st and (k < 4 or st & {10, 12})
    rows = {bytes(r) for r in want.data128}
    assert all(sum(d in rows for d in s) >= 2 for s in sets)             # every committee votes for at least two colliding data
    eng.tree_load(*tree, np.ones(len(tree[0]), np.uint8))
    _intake_both(eng, wires, off, 2, 2, stride, want)


# ------------------------------------------------------------------------------------------ B: the aggregate intake
def _agg_dev(e, members, off, wires):
    """the device form into sentinel-padded views; the outputs as the host form returns them"""
    n, stride = len(wires), G.STRIDE
    wire, woff = _wire(wires)
    t = lambda a: torch.as_tensor(np.ascontiguousarray(a).view(np.int32), device=DEV)      # noqa: E731
    i32 = dict(dtype=torch.int32)
    o = dict(status=_Padded(n, **i32), committee=_Padded(n, **i32), data_id=_Padded(n, **i32), bits=_Padded(n, (stride,)),
             sigs=_Padded(n, (96,)), msgs=_Padded(n, (32,)), target_epoch=_Padded(n, dtype=torch.int64), block_idx=_Padded(n, **i32),
             members=_Padded(n, (8 * stride,), **i32), item_off=_Padded(n + 1, **i32))
    e.aggregate_and_proof_intake_dev(torch.as_tensor(np.frombuffer(wire, np.uint8).copy(), device=DEV), t(woff), t(members), t(off), EPOCH,
                                     G.CUR, G.DOMAINS, G.CPS, G.SPE, *[x.t for x in o.values()], G.TARGET, G.RANGE)
    torch.cuda.synchronize()
    for name, x in o.items():
        assert x.unchanged_outside(0, x.n), name
    r = {name: x.numpy() for name, x in o.items()}
    for name in ("committee", "data_id", "block_idx", "members", "item_off"):
        r[name] = r[name].view(np.uint32)
    r["target_epoch"] = r["target_epoch"].view(np.uint64)
    return types.SimpleNamespace(**r)


def _agg_both(e, members, off, wires, ok, tree):
    """both forms against the oracle on tree (parent, slot, roots), which the engine holds; returns the oracle's result"""
    o = AO.validate(wires, members, off, EPOCH, G.CUR, G.DOMAINS, G.CPS, G.SPE, G.STRIDE, *tree, lambda i: ok[i], G.TARGET, G.RANGE)
    G._same(G._host_call(e, members, off, wires), o)
    G._same(_agg_dev(e, members, off, wires), o)
    assert e.guard_flags() == 0
    return o


G_TREE = (G.PARENT, G.SLOT, G.ROOTS)


def _failing_item(rng, kind, i, fp, lanes=(14, 15)):
    """(aggregator, bits, data) of an item that decodes and fails check kind (4-9), its data on fingerprint fp: word lanes[0] = i, word
    lanes[1] the fix (by default the source root's words 14 and 15)"""
    slot, index, tep, bits = 14, 0, 3, [bool(b) for b in rng.integers(0, 2, G.SIZES[4])]
    if kind == 4:
        index = G.CPS
    elif kind == 5:
        slot = 15                                   # after the current slot
    elif kind == 6:
        slot, tep = 13, 2                           # the target epoch is not the slot's
    elif kind == 7:
        slot, tep = 10, 2                           # another epoch
    elif kind == 8:
        bits = bits + [True]                        # one bit longer than committee 4
    else:
        bits = [False] * G.SIZES[4]                 # no bit
    d = K._set_word(make_data(slot, index, bytes(G.ROOTS[4]), 2, bytes(32), tep, bytes(G.ROOTS[3])), lanes[0], i)
    return int(rng.integers(G.N_VAL)), bits, K.with_fingerprint(d, fp, lanes[1])


def _unsigned(agg, bits, d, rng):
    return AO.encode(agg, bits, d, bytes(96), rng.integers(0, 256, 96, dtype=np.uint8).tobytes(), bytes(96))


def _signed_trio(env, fp, c=0):
    """A: accepted, data X on fingerprint fp, bits S; B: colliding X', bits within S, another aggregator: accepted; C: X, bits within S:
    check 10.  (wires, verdicts)"""
    e, sks, members, off = env
    b = G.Builder(e, sks, members, off)
    a0 = b.aggregator(c)
    a1 = b.aggregator(c, skip=(a0,))
    a2 = b.aggregator(c, skip=(a0, a1))
    n0 = G.SIZES[c]
    b.add(c, [j < n0 // 2 for j in range(n0)], a0)
    x = K.with_fingerprint(b.specs[0]["d"], fp, 20)
    x2 = K.collide(x, 14, 15)
    b.add(c, [j < n0 // 4 for j in range(n0)], a1)
    b.add(c, [j == 1 for j in range(n0)], a2)
    for s, d in zip(b.specs, (x, x2, x)):
        s["d"] = d
    return b.build()


def _table(n):
    tab = 1
    while tab < 2 * n:
        tab <<= 1
    return tab


def _probe_batch(env, n, one_fp, seed):
    """n items for a data table of _table(n) slots: half the failing items on fingerprints = tab - 1 (mod tab), a quarter of those on
    one 32-bit fingerprint, the rest spread; or (one_fp) every item on one fingerprint.  Byte-equal copies of cluster items come last;
    from n = 64 on, the signed trio sits in the middle on the cluster's fingerprint.  (wires, verdicts, cluster fingerprint)"""
    rng = np.random.default_rng(seed)
    mask = _table(n) - 1
    f0 = (0x5A5A5A5A | mask) & K.M32
    n_dup = max(1, n // 4) if n > 1 else 0
    trio = n >= 64
    n_base = n - n_dup - (3 if trio else 0)
    cluster = n_base if one_fp else (n_base + 1) // 2
    items = []
    for i in range(n_base):
        if i >= cluster:
            fp = int(rng.integers(0, 1 << 32))
        elif one_fp or i % 4 == 0:
            fp = f0
        else:
            fp = (int(rng.integers(0, 1 << 32)) | mask) & K.M32
        items.append(_failing_item(rng, 4 + i % 6, i + 1, fp))
    clustered = [it for it in items if (K.fingerprint(it[2]) & mask) == mask]
    dups = [(int(rng.integers(G.N_VAL)), it[1], it[2]) for it in (clustered[-1 - j % len(clustered)] for j in range(n_dup))]
    wires = [_unsigned(a, bits, d, rng) for a, bits, d in items]
    ok = [NO_SIG] * len(wires)
    if trio:
        tw, tok = _signed_trio(env, f0)
        h = len(wires) // 2
        wires, ok = wires[:h] + tw + wires[h:], ok[:h] + tok + ok[h:]
    wires += [_unsigned(a, bits, d, rng) for a, bits, d in dups]
    ok += [NO_SIG] * n_dup
    assert len(wires) == n
    return wires, ok, f0


@pytest.mark.parametrize("n,one_fp", [(1, False), (2, False), (3, False), (64, False), (65, False), (4096, False), (4096, True)])
def test_aggregate_data_table(agg, n, one_fp):
    e, sks, members, off = agg
    e.tree_load(*G_TREE, np.ones(6, np.uint8))
    wires, ok, f0 = _probe_batch(agg, n, one_fp, 7 * n + one_fp)
    fps = [K.fingerprint(bytes(w[AO.ATT + 4:AO.ATT + 132])) for w in wires]
    mask = _table(n) - 1
    assert sum((f & mask) == mask for f in fps) >= max(1, n // 2) and (not one_fp or set(fps) == {f0})
    o = _agg_both(e, members, off, wires, ok, G_TREE)
    st = o.status.tolist()
    assert set(st) >= ({4, 5, 6, 7, 8, 9} if n >= 6 else {4 + i for i in range(n - (n > 1))})
    data = [bytes(w[AO.ATT + 4:AO.ATT + 132]) for w in wires]
    assert len(set(data)) < n or n == 1                                    # byte-equal copies share a data id ...
    assert len(set(o.data_id.tolist())) == len(set(data))                  # ... and distinct data on one fingerprint do not
    if n >= 64:
        h = (n - max(1, n // 4) - 3) // 2
        assert st[h:h + 3] == [0, 0, 10]
        assert o.data_id[h + 2] == o.data_id[h] != o.data_id[h + 1]


# ------------------------------------------------------------------------------------------ C: roots
SPE_C, CPS_C, STRIDE_C = G.SPE, G.CPS, 128      # the aggregate world's epoch layout: slots 12 .. 15, the current slot 14 for gossip
START = EPOCH * SPE_C


def _root_world(seed=5):
    """ids 0 (slot 9), 1 = the anchor (slot 12, start of the epoch), 2 (slot 10, a branch the prune drops), one hub per group (slot 13,
    under the anchor), the groups' roots as leaves under their hubs (slot 14) in random id order.  The tree holds 00..00, below which no
    root lies, and ff..fe, above which only ff..ff lies: the tests name ff..ff as head and target (it is no tree root, only the oracle's
    parent of block 0), so that the root search's exit past the last sorted id runs in every form, not only on the one-block tree."""
    rng = np.random.default_rng(seed)
    groups = list(K.shared_prefix_groups(rng).values()) + [list(p) for p in K.le_flip_pairs(rng)] + [K.edge_roots()]
    fixed = [bytes(r) for r in rng.integers(0, 255, (3 + len(groups), 32), dtype=np.uint8)]
    leaves = [(g, r) for g, grp in enumerate(groups) for r in grp]
    leaves = [leaves[i] for i in rng.permutation(len(leaves))]
    hubs = list(range(3, 3 + len(groups)))
    parent = [0, 0, 0] + [1] * len(groups) + [hubs[g] for g, _ in leaves]
    slot = [9, 12, 10] + [13] * len(groups) + [14] * len(leaves)
    roots = fixed + [r for _, r in leaves]
    assert len(set(roots)) == len(roots) and K.OUTSIDE not in roots
    return np.array(parent, np.uint32), np.array(slot, np.uint64), np.frombuffer(b"".join(roots), np.uint8).reshape(-1, 32).copy(), hubs


def _tree_form(e, form):
    """(parent, slot, roots, hubs, anchor) after building the world on the device as `form`"""
    if form == "one_block":
        root = bytes(range(0x70, 0x90))
        e.tree_load([0], [START], np.frombuffer(root, np.uint8).reshape(1, 32), [1])
        return np.zeros(1, np.uint32), np.array([START], np.uint64), np.frombuffer(root, np.uint8).reshape(1, 32), [], 0
    parent, slot, roots, hubs = _root_world()
    n, n0 = len(parent), 3 + len(hubs)
    if form == "loaded":
        e.tree_load(parent, slot, roots, np.ones(n, np.uint8))
        return parent, slot, roots, hubs, 1
    e.tree_load(parent[:n0], slot[:n0], roots[:n0], np.ones(n0, np.uint8))
    j = n0
    for size in [1] * 5 + [3, 7, 2, n]:           # one at a time, then batches whose roots interleave with the tree's
        k = min(size, n - j)
        if k == 0:
            break
        e.tree_add(parent[j:j + k], slot[j:j + k], roots[j:j + k], np.ones(k, np.uint8))
        j += k
    assert e.tree_size() == n
    if form == "added":
        return parent, slot, roots, hubs, 1
    model = TU.Model(parent, roots, np.ones(n, np.uint8), 8)
    mp = e.tree_prune(1)                           # the anchor becomes block 0; blocks 0 and 2 leave the tree
    assert np.array_equal(mp, model.prune(1))
    return model.parent, slot[mp != NONE], model.roots, [int(mp[h]) for h in hubs], 0


def _intake_roots(rng, tree, anchor, valid_head, gone=()):
    """the intake's wires: every root as head (target the anchor) and as target (head valid_head) in the committees of slot 15; every
    one-byte neighbour of every root, every root in `gone` and ff..ff, as head in those of slots 12 and 13, and as target in those of
    slots 14 and 15.  Returns (wires, off, expectations: (list index, status or None, block id or None, committee, position))"""
    _, _, roots = tree
    rl = [bytes(r) for r in roots]
    size = 8 * STRIDE_C
    free = {c: list(range(size)) for c in range(SPE_C * CPS_C)}
    items, expect = [], []

    def put(cs, head, target, status, blk=None):
        c = max(cs, key=lambda q: len(free[q]))
        p = free[c].pop(int(rng.integers(len(free[c]))))
        expect.append((len(items), status, blk, c, p))
        items.append((c, p, make_data(START + c // CPS_C, c % CPS_C, head, EPOCH - 1, bytes(32), EPOCH, target)))

    for b, r in enumerate(rl):
        put([6, 7], r, rl[anchor], None, b)
        put([6, 7], rl[valid_head], r, 0 if b == anchor else 12)
        for m in K.near_misses(r, rl):
            put([0, 1, 2, 3], m, rl[anchor], 9)
            put([4, 5, 6, 7], rl[valid_head], m, 10)
    for r in list(gone) + [K.OUTSIDE]:                 # ff..ff: above every root of the tree
        put([0, 1, 2, 3], r, rl[anchor], 9)
        put([4, 5, 6, 7], rl[valid_head], r, 10)
    order = rng.permutation(len(items))
    pos = np.argsort(order)
    wires = [_att(size, items[i][1], items[i][2], rng) for i in order]
    return wires, IO.ragged_layout([size] * SPE_C * CPS_C), [(int(pos[i]), s, b, c, p) for i, s, b, c, p in expect]


def _gossip_roots(env, rng, tree, anchor, valid_head):
    """gossip items of committee 4 (slot 14) with an empty bit row (check 9, block_idx still looked up): every root, every one-byte
    neighbour and ff..ff as head; then three signed items: a found head (accepted), an unknown head (17), an unknown target (18)"""
    e, sks, members, off = env
    rl = [bytes(r) for r in tree[2]]
    heads = [(r, b) for b, r in enumerate(rl)] + [(m, NONE) for r in rl for m in K.near_misses(r, rl)] + [(K.OUTSIDE, NONE)]
    wires = []
    for i, (h, _) in enumerate(heads):
        d = K._set_word(make_data(14, 0, h, 2, bytes(32), 3, rl[anchor]), 14, i + 1)
        wires.append(_unsigned(int(rng.integers(G.N_VAL)), [False] * G.SIZES[4], d, rng))
    b = G.Builder(e, sks, members, off)
    aggs = []
    for _ in range(3):
        aggs.append(b.aggregator(4, skip=tuple(aggs)))
    full = [True] * G.SIZES[4]
    b.add(4, full, aggs[0], head_root=rl[valid_head], target_root=rl[anchor])
    b.add(4, full, aggs[1], head_root=K.near_miss(rl[valid_head], 31, 1), target_root=rl[anchor])
    b.add(4, full, aggs[2], head_root=rl[valid_head], target_root=K.near_miss(rl[anchor], 16, -1))
    sw, sok = b.build()
    return wires + sw, [NO_SIG] * len(wires) + sok, [blk for _, blk in heads]


@pytest.mark.parametrize("form", ["loaded", "added", "pruned", "one_block"])
def test_roots(agg, form):
    e, sks, members, off = agg
    rng = np.random.default_rng(len(form))
    e.latest_messages_reset()
    parent, slot, roots, hubs, anchor = _tree_form(e, form)
    tree = (parent, slot, roots)
    n = len(parent)
    valid_head = n - 1 if n > 1 else 0                  # a leaf (slot 14) under the anchor
    assert int(slot[valid_head]) <= 14 and IO.ancestor(parent, slot, valid_head, START) == anchor
    # the attestation intake: statuses 9 and 10 for the neighbours, block ids for the roots
    gone = [bytes(r) for r in _root_world()[2][[0, 2]]] if form == "pruned" else []      # the blocks the prune dropped
    wires, aoff, expect = _intake_roots(rng, tree, anchor, valid_head, gone)
    want = _numpy_oracle(tree, wires, aoff, SPE_C, CPS_C, STRIDE_C)
    for i, status, blk, c, p in expect:
        if status is not None:
            assert want.status[i] == status, (i, status, int(want.status[i]))
        if blk is not None and want.status[i] == 0:
            assert want.block_idx[want.vote[int(aoff[c]) + p]] == blk
    assert sum(1 for i, s, b, c, p in expect if b is not None and want.status[i] == 0) >= (len(hubs) + 1 if n > 1 else 1)
    _intake_both(e, wires, aoff, SPE_C, CPS_C, STRIDE_C, want)
    # the aggregate intake: block_idx of every head, 17 and 18 for the signed neighbours
    gw, gok, blk = _gossip_roots(agg, rng, tree, anchor, valid_head)
    o = _agg_both(e, members, off, gw, gok, tree)
    assert o.block_idx[:len(blk)].tolist() == blk
    assert o.status[-3:].tolist() == [0, 17, 18]
    # get_head: the tied fan of every group (no votes), at the root and at every hub
    model = TU.Model(parent, roots, np.ones(n, np.uint8), 8)
    ref = TU.engine(model)
    TU.load(ref, model)
    for j in [0] + hubs:
        assert e.get_head(j) == ref.get_head(j) == model.head(j), j
    ref.close()


# ------------------------------------------------------------------------------------------ D: one committee flooded
def _timed(fn, reps=3):
    """wall time of fn() up to a device synchronise, after one warm-up call: 'median (min - max) ms' of reps calls"""
    fn()
    torch.cuda.synchronize()
    ms = []
    for _ in range(reps):
        t = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ms.append(1e3 * (time.perf_counter() - t))
    ms.sort()
    return "%.1f ms (%.1f - %.1f)" % (ms[len(ms) // 2], ms[0], ms[-1])


@pytest.mark.parametrize("one_fp", [False, True])
def test_intake_flood_one_committee(eng, one_fp):
    """8 192 attestations, four per member of one 2 048-member committee, each with its own datum (a seventh with an unknown target, at
    most one per member); on spread fingerprints or all on one.  The data differ first in word 20 (bytes 80..83, the source root), with
    word 21 the fix: the latest two valid attestations can differ, so that every byte comparison runs past byte 80."""
    rng = np.random.default_rng(60 + one_fp)
    size, n = 2048, 8192
    tree = (np.array([0, 0], np.uint32), np.array([0, EPOCH], np.uint64), np.array([[7] * 32, [9] * 32], np.uint8))
    x = make_data(EPOCH, 0, bytes([9] * 32), EPOCH - 1, bytes([7] * 32), EPOCH, bytes([9] * 32))
    variants = []
    for i in range(1, n):
        v = K._set_word(x, 20, K._word(x, 20) ^ i)
        variants.append(K._set_word(v, 31, K._word(v, 31) ^ i) if i % 7 == 3 else v)
    data = K.collision_set(x, variants, 21) if one_fp else [x] + variants
    assert len(set(data)) == n and (len({K.fingerprint(d) for d in data}) == 1) == one_fp
    wires = [_att(size, a % size, data[a], rng) for a in rng.permutation(n)]
    off = IO.ragged_layout([size])
    want = _numpy_oracle(tree, wires, off, 1, 1, 256)
    assert set(want.status.tolist()) == {0, 10, 13} and int(want.vote_off[-1]) == size
    eng.tree_load(*tree, np.ones(2, np.uint8))
    _intake_both(eng, wires, off, 1, 1, 256, want)
    wire, woff = _wire(wires)
    d_wire, d_woff = torch.as_tensor(np.frombuffer(wire, np.uint8).copy(), device=DEV), torch.as_tensor(woff.view(np.int32), device=DEV)
    d_off = torch.as_tensor(off.view(np.int32), device=DEV)
    z = lambda *s, dt=torch.int32: torch.zeros(*s, dtype=dt, device=DEV)      # noqa: E731
    outs = (z(n), z(size), z(2), z((size, 96), dt=torch.uint8), z((size, 128), dt=torch.uint8), z((size, 32), dt=torch.uint8),
            z(size, dt=torch.int64), z(size, dt=torch.int64), z(size))
    ms = _timed(lambda: eng.attestation_intake_dev(d_wire, d_woff, d_off, EPOCH, EPOCH + 1, DOMAIN, 1, 1, 256, *outs))
    print("attestation intake, 8192 attestations in one 2048-member committee%s: %s" % (" on one fingerprint" if one_fp else "", ms))


def test_aggregate_flood_one_committee(agg):
    """2 048 aggregates of committee 3 (31 members): the signed trio first, then unsigned items of mostly other aggregators (12 or 13;
    14 where an unsigned item passes both), a few shadowed by the accepted item (10) or of its aggregator (11)"""
    e, sks, members, off = agg
    e.tree_load(*G_TREE, np.ones(6, np.uint8))
    rng = np.random.default_rng(70)
    n = 2048
    tw, tok = _signed_trio(agg, FP, 3)
    com = G._committee(members, off, 3)
    x = make_data(13, 1, bytes(G.ROOTS[4]), 2, bytes(32), 3, bytes(G.ROOTS[3]))
    wires = []
    for i in range(n - 3):
        d = K.with_fingerprint(K._set_word(x, 14, i % 64), FP, 15)
        a = com[int(rng.integers(len(com)))] if rng.random() < 0.9 else int(rng.integers(G.N_VAL))
        bits = [bool(b) for b in rng.integers(0, 2, len(com))]
        bits[int(rng.integers(len(com)))] = True
        wires.append(_unsigned(a, bits, d, rng))
    wires, ok = tw + wires, tok + [NO_SIG] * (n - 3)
    o = _agg_both(e, members, off, wires, ok, G_TREE)
    st = np.bincount(o.status, minlength=21)
    assert st[12] + st[13] > n // 2 and st[0] >= 2 and st[10] >= 1, st.tolist()
    wire, woff = _wire(wires)
    d_wire, d_woff = torch.as_tensor(np.frombuffer(wire, np.uint8).copy(), device=DEV), torch.as_tensor(woff.view(np.int32), device=DEV)
    t = lambda a: torch.as_tensor(np.ascontiguousarray(a).view(np.int32), device=DEV)      # noqa: E731
    z = lambda *s, dt=torch.int32: torch.zeros(*s, dtype=dt, device=DEV)                    # noqa: E731
    outs = (z(n), z(n), z(n), z((n, G.STRIDE), dt=torch.uint8), z((n, 96), dt=torch.uint8), z((n, 32), dt=torch.uint8), z(n, dt=torch.int64),
            z(n), z((n, 8 * G.STRIDE)), z(n + 1))
    dm, do = t(members), t(off)
    ms = _timed(lambda: e.aggregate_and_proof_intake_dev(d_wire, d_woff, dm, do, EPOCH, G.CUR, G.DOMAINS, G.CPS, G.SPE, *outs, G.TARGET, G.RANGE))
    print("aggregate intake, 2048 items in one committee: %s" % ms)


def test_aggregate_one_fingerprint_timing(agg):
    """the device time of 4 096 failing items on one fingerprint against the same batch on spread fingerprints.  The data differ only in
    the target root's last two words (30 = the item, 31 = the fix), so every compare of the up to 4 096-long probe chains reads 121 to
    124 bytes."""
    e, sks, members, off = agg
    e.tree_load(*G_TREE, np.ones(6, np.uint8))
    res = {}
    for one_fp in (False, True):
        rng = np.random.default_rng(80)
        items = [_failing_item(rng, 9, i + 1, FP if one_fp else int(rng.integers(0, 1 << 32)), (30, 31)) for i in range(4096)]
        wires = [_unsigned(a, bits, d, rng) for a, bits, d in items]
        n = len(wires)
        wire, woff = _wire(wires)
        d_wire, d_woff = torch.as_tensor(np.frombuffer(wire, np.uint8).copy(), device=DEV), torch.as_tensor(woff.view(np.int32), device=DEV)
        t = lambda a: torch.as_tensor(np.ascontiguousarray(a).view(np.int32), device=DEV)      # noqa: E731
        z = lambda *s, dt=torch.int32: torch.zeros(*s, dtype=dt, device=DEV)                    # noqa: E731
        outs = (z(n), z(n), z(n), z((n, G.STRIDE), dt=torch.uint8), z((n, 96), dt=torch.uint8), z((n, 32), dt=torch.uint8),
                z(n, dt=torch.int64), z(n), z((n, 8 * G.STRIDE)), z(n + 1))
        dm, do = t(members), t(off)
        res[one_fp] = _timed(lambda: e.aggregate_and_proof_intake_dev(d_wire, d_woff, dm, do, EPOCH, G.CUR, G.DOMAINS, G.CPS, G.SPE, *outs,
                                                                      G.TARGET, G.RANGE))
        assert (outs[0].cpu().numpy() == 9).all() and len(set(outs[2].cpu().numpy().tolist())) == n
    print("aggregate intake, 4096 items: %s on spread fingerprints, %s on one fingerprint" % (res[False], res[True]))


# ------------------------------------------------------------------------------------------ E: end to end
def test_colliding_votes_end_to_end(eng):
    """committee 0 split between X and a colliding X' (both valid), committee 1 on Y; signed with the members' keys"""
    from pos_evolution_b200.epoch import EpochProcessor
    rng = np.random.default_rng(21)
    spe, cps, stride, sizes = 2, 1, 8, [64, 40]
    n_val = sum(sizes)
    tree = IO.random_tree(rng, 12, EPOCH * spe - 3)
    parent, slot, roots = tree
    start = EPOCH * spe
    members = rng.permutation(n_val).astype(np.uint32)
    off = IO.ragged_layout(sizes)
    eff = rng.integers(16, 33, n_val).astype(np.uint64) * np.uint64(10**9)
    eng.registry_load(np.frombuffer(b"".join(scenarios.pubkeys(n_val)), np.uint8), eff)
    eng.tree_load(*tree, np.ones(len(parent), np.uint8))
    eng.latest_messages_reset()
    data = []
    for c in range(2):
        h = _good_heads(tree, start + c, start)[-1]
        data.append(make_data(start + c, 0, bytes(roots[h]), EPOCH - 1, bytes(roots[0]), EPOCH, bytes(roots[IO.ancestor(parent, slot, h, start)])))
    x, y = data
    x2 = K.collide(x, 14, 15)
    per = [(0, p, x2 if p % 3 == 1 else x) for p in range(sizes[0]) if p % 7 != 3] + [(1, p, y) for p in range(sizes[1])]
    per = [per[i] for i in rng.permutation(len(per))]
    datas = [x, x2, y]
    msgs = np.frombuffer(b"".join(Spec.compute_signing_root(IO.data_from_bytes(d), DOMAIN) for d in datas), np.uint8).reshape(3, 32)
    sig = eng.sign([scenarios.secret_key(int(members[off[c] + p])) for c, p, _ in per], [datas.index(d) for _, _, d in per], msgs)
    wires = [IO.encode([j == p for j in range(sizes[c])], d, bytes(sig[a])) for a, (c, p, d) in enumerate(per)]
    r = IO.intake_plain(wires, off, EPOCH, (EPOCH + 1) * spe, DOMAIN, cps, spe, stride, *IO.block_store(*tree))
    assert (r.status == 0).all() and r.vote_off.tolist() == [0, 2, 3]
    assert sorted(bytes(d) for d in r.data128[:2]) == sorted([x, x2])
    ep = EpochProcessor(eng, 2, n_val, stride, len(parent), device=DEV, depth=2, max_votes=4)
    ep.set_committees(members, off)
    wire, woff = _wire(wires)
    with torch.cuda.stream(torch.cuda.Stream()):
        xi = ep.intake_dev(torch.as_tensor(np.frombuffer(wire, np.uint8).copy(), device=DEV), torch.as_tensor(woff.view(np.int32), device=DEV),
                           EPOCH, (EPOCH + 1) * spe, DOMAIN, cps, spe)
    assert np.array_equal(xi.status.cpu().numpy(), r.status) and np.array_equal(xi.vote_off, r.vote_off)
    assert np.array_equal(xi.vote.cpu().numpy().view(np.uint32), r.vote)
    ok, hd = ep.process_epoch_dev(xi.sigs, None, xi.msgs, xi.target_epoch, xi.block_idx, votes=(xi.vote, xi.vote_off))
    torch.cuda.synchronize()
    assert ok.cpu().numpy().tolist() == [1, 1, 1]
    agg_sig = ep.slots[0].agg_sig[:3].cpu().numpy()
    m_epoch, m_block, m_has = np.zeros(n_val, np.uint64), np.zeros(n_val, np.uint32), np.zeros(n_val, np.uint8)
    equiv = np.zeros(n_val, np.uint8)
    com = np.repeat(np.arange(2), sizes)
    for v in range(3):
        slots_v = np.nonzero(r.vote == v)[0]
        who = members[slots_v].tolist()
        assert bytes(agg_sig[v]) == scenarios.sign_aggregate(who, bytes(r.msgs[v])), v
        assert (com[slots_v] == (v == 2)).all()
        fast.lmd_update(m_epoch, m_block, m_has, equiv, who, int(r.target_epoch[v]), int(r.block_idx[v]))
    w = fast.ghost_weights(parent, m_block, m_has, eff, np.ones(n_val, np.uint8), equiv, -1, 0)
    assert int(hd.item()) == fast.ghost_head(parent, roots, fast.ghost_viable(parent, np.ones(len(parent), np.uint8)), w, 0)
    e_, b_, h_ = eng.latest_messages_read()
    assert np.array_equal(h_, m_has) and np.array_equal(e_[h_ == 1], m_epoch[h_ == 1]) and np.array_equal(b_[h_ == 1], m_block[h_ == 1])
