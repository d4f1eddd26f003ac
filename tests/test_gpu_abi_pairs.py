"""Both forms of every C-ABI entry point that comes as a host form (b2_X) and a device form (b2_X_dev) reject the same arguments alike.

Each pair starts from one small valid argument set, which both forms accept.  Each mutation then breaks exactly one condition on the
arguments both forms receive (a zero count, a bits_stride of 0 or 257, a committee count that does not match, an epoch outside the
window, a null pointer, ...) and both forms are called with outputs the test owns, filled with a sentinel: numpy arrays for the host
form, CUDA tensors for the device form.  Both calls must return B2_EINVAL with the same b2_last_error text, launch nothing, leave every
output byte as it was and leave the device tables (latest messages, both participation tables, weights, head, equivocating) answering
as before.  The loaded-state preconditions (no registry, tree, slasher, sync committee or participation tables) run on fresh engines."""
import numpy as np
import pytest
import torch

import aggregate_intake_oracle as AIO
import block_attestations_electra_oracle as BAE
import intake_oracle as IO
import scenarios
import sync_messages_oracle as SM

pytestmark = pytest.mark.gpu

SENTINEL = 0xA5
N_VAL, N_BLK, N_AGG, CSIZE = 64, 40, 4, 8
EPOCH, SPE = 3, 4
CUR_SLOT = EPOCH * SPE + 1
MSG = np.arange(32, dtype=np.uint8).reshape(1, 32)


class In:
    """an input array: the host form gets it as is, the device form a copy in device memory"""
    def __init__(self, a):
        self.a = np.ascontiguousarray(a)


class HostIn(In):
    """an array both forms read from host memory (the domains and the justified checkpoint)"""


class Out:
    """an output of n bytes, sentinel-filled"""
    def __init__(self, n):
        self.n = n


class DevOnly:
    """a count only the device form takes; the host form derives it from its offsets"""
    def __init__(self, v):
        self.v = v


def _bytes(*arrays):
    return np.frombuffer(b"".join(bytes(a) for a in arrays), np.uint8)


def _batch():
    members = np.arange(N_AGG * CSIZE, dtype=np.uint32) % N_VAL
    off = np.arange(0, (N_AGG + 1) * CSIZE, CSIZE, dtype=np.uint32)
    return members, off, np.full((N_AGG, CSIZE // 8), 0xFF, np.uint8)


def _wire(wires):
    return In(_bytes(*wires)), sum(len(w) for w in wires), In(np.cumsum([0] + [len(w) for w in wires]).astype(np.uint32))


def _data128(roots):
    return IO.data128(EPOCH * SPE, 0, bytes(roots[1]), EPOCH - 1, bytes(32), EPOCH, bytes(roots[0]))


# Each pair: its arguments in the order of the host form's parameters (a DevOnly one sits where the device form takes it), the mutations
# {label: {argument: new value}} on top of a null for every pointer not in `optional`, and the arguments that may be null.
def _aggregate(eng, roots):
    sigs = eng.sign([1, 2, 3, 4], [0, 0, 0, 0], MSG)
    args = dict(sig96=In(sigs), seg_off=In(np.array([0, 2, 4], np.uint32)), n_seg=2, n_sig=DevOnly(4), out96=Out(2 * 96), seg_status=Out(2 * 4))
    return args, {"n_seg=0": dict(n_seg=0)}, ()


def _fast_aggregate_verify(eng, roots):
    members, off, bits = _batch()
    args = dict(members=In(members), off=In(off), bits=In(bits), bits_stride=1, msg32=In(np.repeat(MSG, N_AGG, 0)),
                sig96=In(eng.sign([1] * N_AGG, [0] * N_AGG, MSG)), n_agg=N_AGG, ok_out=Out(N_AGG))
    return args, {"n_agg=0": dict(n_agg=0), "bits_stride=0": dict(bits_stride=0)}, ()


def _aggregate_verify(eng, roots):
    args = dict(signer=In(np.arange(4, dtype=np.uint32)), msg32=In(np.repeat(MSG, 4, 0)), pair_off=In(np.array([0, 2, 4], np.uint32)),
                n_pairs=DevOnly(4), sig96=In(eng.sign([3, 7], [0, 0], MSG)), n_sets=2, ok_out=Out(2))
    too_many = dict(pair_off=In(np.array([0, 2, 0xFFFFFFFF], np.uint32)), n_pairs=DevOnly(0xFFFFFFFF))
    return args, {"n_sets=0": dict(n_sets=0), "n_pairs + n_sets >= 2^32": too_many}, ()


def _sync_aggregate_verify(eng, roots):
    args = dict(committee_idx=In(np.zeros(2, np.uint32)), bits=In(np.full((2, 2), 0x0F, np.uint8)), msg32=In(np.repeat(MSG, 2, 0)),
                sig96=In(eng.sign([10, 20], [0, 0], MSG)), n=2, ok_out=Out(2), pk48_out=Out(2 * 48))
    return args, {"n=0": dict(n=0)}, ("pk48_out",)


def _attestation_intake(eng, roots):
    wires = [IO.encode([True] * CSIZE, _data128(roots), bytes(96)), IO.encode([i == 2 for i in range(CSIZE)], _data128(roots), bytes(96))]
    wire, wire_len, woff = _wire(wires)
    n_c, n_sig, mv = SPE, SPE * CSIZE, 16
    args = dict(wire=wire, wire_len=wire_len, woff=woff, n_att=2, off=In(np.arange(0, n_sig + 1, CSIZE, dtype=np.uint32)), n_committees=n_c,
                n_sig=DevOnly(n_sig), committees_per_slot=1, slots_per_epoch=SPE, bits_stride=1, epoch=EPOCH, current_slot=CUR_SLOT,
                domain32=HostIn(np.full(32, 7, np.uint8)), max_votes=mv, status_out=Out(4 * 2), vote_out=Out(4 * n_sig),
                vote_off_out=Out(4 * (n_c + 1)), sig96_out=Out(96 * n_sig), data128_out=Out(128 * mv), msg32_out=Out(32 * mv),
                source_epoch_out=Out(8 * mv), target_epoch_out=Out(8 * mv), block_idx_out=Out(4 * mv))
    return args, {"n_att=0": dict(n_att=0), "max_votes=0": dict(max_votes=0), **_intake_mutations()}, ()


def _intake_mutations():
    return {"bits_stride=0": dict(bits_stride=0), "bits_stride=257": dict(bits_stride=257), "committees_per_slot=0": dict(committees_per_slot=0),
            "slots_per_epoch=0": dict(slots_per_epoch=0), "n_committees wrong": dict(n_committees=SPE - 1),
            "epoch two ahead": dict(epoch=EPOCH + 2), "epoch behind the window": dict(epoch=EPOCH - 2), "current_slot >= 2^63": dict(current_slot=1 << 63)}


def _aggregate_and_proof_intake(eng, roots):
    wires = [AIO.encode(v, [True] * CSIZE, _data128(roots), bytes(96), bytes(96), bytes(96)) for v in (0, 9)]
    wire, wire_len, woff = _wire(wires)
    n, n_sig, members = 2, SPE * CSIZE, np.arange(SPE * CSIZE, dtype=np.uint32) % N_VAL
    args = dict(wire=wire, wire_len=wire_len, woff=woff, n=n, members=In(members), off=In(np.arange(0, n_sig + 1, CSIZE, dtype=np.uint32)),
                n_committees=SPE, n_sig=DevOnly(n_sig), committees_per_slot=1, slots_per_epoch=SPE, bits_stride=1, epoch=EPOCH,
                current_slot=CUR_SLOT, domains96=HostIn(np.full(96, 5, np.uint8)), target_aggregators=16, propagation_slot_range=32,
                status_out=Out(4 * n), committee_out=Out(4 * n), data_id_out=Out(4 * n), bits_out=Out(n), sig96_out=Out(96 * n), msg32_out=Out(32 * n),
                target_epoch_out=Out(8 * n), block_idx_out=Out(4 * n), members_out=Out(4 * n * 8), item_off_out=Out(4 * (n + 1)))
    bad = {"n=0": dict(n=0), "n=2^28": dict(n=1 << 28), "n * 8 * bits_stride >= 2^32": dict(n=1 << 21, bits_stride=256),
           "target_aggregators=0": dict(target_aggregators=0), **_intake_mutations()}
    return args, bad, ()


def _block_attestation_args(wires, roots, shape):
    """both block-attestation calls: two attestations in one block of epoch EPOCH, one committee per slot; `shape` the form's
    member-row arguments, which sit between min_inclusion_delay and effective_balance_increment"""
    wire, wire_len, woff = _wire(wires)
    n_c = 2 * SPE
    n_sig = n_c * CSIZE
    args = dict(wire=wire, wire_len=wire_len, woff=woff, n_att=2, block_off=In(np.array([0, 2], np.uint32)),
                block_slot=In(np.array([EPOCH * SPE + 2], np.uint64)), n_blocks=1, members=In(np.arange(n_sig, dtype=np.uint32) % N_VAL),
                off=In(np.arange(0, n_sig + 1, CSIZE, dtype=np.uint32)), n_committees=n_c, n_sig=DevOnly(n_sig), cps_prev=1, cps_cur=1,
                chain_roots=In(np.tile(roots[:2].reshape(1, 64), (SPE, 1))), justified80=HostIn(np.zeros(80, np.uint8)),
                domains64=HostIn(np.full(64, 3, np.uint8)), slots_per_epoch=SPE, min_inclusion_delay=1, **shape,
                effective_balance_increment=10**9, base_reward_per_increment=100, status_out=Out(4 * 2), flag_mask_out=Out(2),
                numerator_out=Out(8 * 2), block_status_out=Out(4), block_first_out=Out(4), block_reward_out=Out(8), n_applied_out=Out(4))
    bad = {"n_att=0": dict(n_att=0), "n_att=2^28": dict(n_att=1 << 28), "n_blocks=0": dict(n_blocks=0), "slots_per_epoch=0": dict(slots_per_epoch=0),
           "cps_cur=0": dict(cps_cur=0), "min_inclusion_delay=0": dict(min_inclusion_delay=0),
           "effective_balance_increment=0": dict(effective_balance_increment=0), "committees >= 2^31": dict(cps_cur=1 << 30),
           "n_committees wrong": dict(n_committees=n_c + 1)}
    return args, bad


def _block_attestations(eng, roots):
    args, bad = _block_attestation_args([IO.encode([True] * CSIZE, _data128(roots), bytes(96))] * 2, roots, dict(bits_stride=1))
    return args, {**bad, "bits_stride=0": dict(bits_stride=0), "bits_stride=257": dict(bits_stride=257)}, ()


def _block_attestations_electra(eng, roots):
    # the device form also takes row_max, which the host form derives from off
    shape = dict(max_committees_per_slot=1, max_validators_per_committee=CSIZE, row_max=DevOnly(CSIZE))
    args, bad = _block_attestation_args([BAE.encode([True] * CSIZE, _data128(roots), bytes(96), [True])] * 2, roots, shape)
    # n_att times the padded row at 2^32 members: one slot of 2 049 members pads to 4 096 (BAE_CHUNK 2 048), 2^20 attestations in one block
    sizes = [CSIZE] * (2 * SPE)
    sizes[SPE + 1] = 2049
    off = np.concatenate([[0], np.cumsum(sizes)]).astype(np.uint32)
    assert BAE.row_max(off, 1, 1, SPE) == 2049
    n_att = 1 << 20
    wide = dict(woff=In(np.zeros(n_att + 1, np.uint32)), n_att=n_att, block_off=In(np.array([0, n_att], np.uint32)),
                members=In(np.arange(off[-1], dtype=np.uint32) % N_VAL), off=In(off), n_sig=DevOnly(int(off[-1])), row_max=DevOnly(2049))
    bad.update({"max_committees_per_slot=0": dict(max_committees_per_slot=0), "max_committees_per_slot=65": dict(max_committees_per_slot=65),
                "max_validators_per_committee=0": dict(max_validators_per_committee=0),
                "M * max_validators_per_committee >= 2^31": dict(max_committees_per_slot=64, max_validators_per_committee=1 << 25),
                "n_att * padded row >= 2^32": wide})
    return args, bad, ()


def _sync_committee_messages(eng, roots):
    size, count, n = 16, 4, 2
    wires = [SM.encode(CUR_SLOT, bytes(roots[0]), v, bytes(96)) for v in (1, 6)]
    wire, wire_len, woff = _wire(wires)
    sub = size // count
    args = dict(wire=wire, wire_len=wire_len, woff=woff, n=n, subnet=In(np.array([0, 1], np.uint32)),
                position_validator=In(np.arange(size, dtype=np.uint32)), committee_size=size, subnet_count=count, current_slot=CUR_SLOT,
                domain32=HostIn(np.full(32, 9, np.uint8)), status_out=Out(4 * n), root_id_out=Out(4 * n), roots32_out=Out(32 * n),
                n_roots_out=Out(4), contrib_bits_out=Out(n * count * ((sub + 7) // 8)), contrib_sig96_out=Out(n * count * 96),
                contrib_present_out=Out(n * count), agg_bits_out=Out(n * ((size + 7) // 8)), agg_sig96_out=Out(n * 96))
    bad = {"n=0": dict(n=0), "n=2^24": dict(n=1 << 24), "committee_size=0": dict(committee_size=0), "subnet_count=0": dict(subnet_count=0),
           "committee_size % subnet_count != 0": dict(subnet_count=3), "committee_size > 1024": dict(committee_size=2048),
           "n * (subnet_count + 1) >= 2^31": dict(n=1 << 23, subnet_count=256, committee_size=512)}
    return args, bad, ()


def _shuffle_committees(eng, roots):
    args = dict(seed32=In(np.arange(32, dtype=np.uint8)), active=None, n_active=10, rounds=10, members_out=Out(4 * 10))
    return args, {"rounds=256": dict(rounds=256)}, ("active",)


def _latest_messages_update(eng, roots):
    members, off, bits = _batch()
    args = dict(members=In(members), off=In(off), bits=In(bits), bits_stride=1, target_epoch=In(np.full(N_AGG, 5, np.uint64)),
                block_idx=In(np.ones(N_AGG, np.uint32)), accept=In(np.ones(N_AGG, np.uint8)), n_agg=N_AGG)
    return args, {"n_agg=0": dict(n_agg=0), "bits_stride=0": dict(bits_stride=0)}, ("accept",)


def _slasher_advance(eng, roots):
    # the host form moves the window to EPOCH + 1, the device form to EPOCH + 1 again (a no-op)
    return dict(current_epoch=EPOCH + 1), {"backwards": dict(current_epoch=EPOCH - 1), "2^32 - 1": dict(current_epoch=0xFFFFFFFF)}, ()


def _slasher_update(eng, roots):
    members, off, bits = _batch()
    total = int(off[-1])
    args = dict(members=In(members), off=In(off), bits=In(bits), bits_stride=1, source_epoch=In(np.full(N_AGG, EPOCH - 1, np.uint64)),
                target_epoch=In(np.full(N_AGG, EPOCH, np.uint64)), data_root32=In(np.tile(roots[2], (N_AGG, 1))), accept=None, n_agg=N_AGG,
                att_status_out=Out(4 * N_AGG), kind_out=Out(total), conflict_target_out=Out(8 * total), n_flagged_out=Out(4))
    return args, {"n_agg=0": dict(n_agg=0), "bits_stride=0": dict(bits_stride=0)}, ("accept", "conflict_target_out")


def _slasher_discount(eng, roots):
    args = dict(members=In(np.arange(6, dtype=np.uint32)), kind=In(np.zeros(6, np.uint8)), n_slots=6, new_out=Out(6), n_new_out=Out(4))
    return args, {"n_slots=0": dict(n_slots=0), "n_slots=2^32": dict(n_slots=1 << 32)}, ()


def _pack_attestations(eng, roots):
    max_out, n_cand = 4, 2
    args = dict(members=In(np.arange(4, dtype=np.uint32)), committee_off=In(np.array([0, 4], np.uint32)), committee_table=In(np.zeros(1, np.uint8)),
                n_committees=1, cand_committee=In(np.zeros(n_cand, np.uint32)), cand_data=In(np.zeros(n_cand, np.uint32)),
                cand_flag_mask=In(np.full(n_cand, 7, np.uint8)), bits=In(np.array([[0x03], [0x0C]], np.uint8)), bits_stride=1,
                sig96=In(eng.sign([1 + 2, 3 + 4], [0, 0], MSG)), n_cand=n_cand, max_out=max_out, effective_balance_increment=10**9,
                base_reward_per_increment=100, n_out=Out(4), out_committee=Out(4 * max_out), out_data=Out(4 * max_out), out_bits=Out(max_out),
                out_sig96=Out(96 * max_out), out_numerator=Out(8 * max_out), out_src_off=Out(4 * (max_out + 1)), out_src=Out(4 * n_cand),
                cand_status=Out(n_cand))
    bad = {"max_out=0": dict(max_out=0), "bits_stride=0": dict(bits_stride=0), "bits_stride=257": dict(bits_stride=257),
           "effective_balance_increment=0": dict(effective_balance_increment=0)}
    return args, bad, ()


PAIRS = {f.__name__[1:]: f for f in (_aggregate, _fast_aggregate_verify, _aggregate_verify, _sync_aggregate_verify, _attestation_intake,
                                     _aggregate_and_proof_intake, _block_attestations, _block_attestations_electra, _sync_committee_messages,
                                     _shuffle_committees,
                                     _latest_messages_update, _slasher_advance, _slasher_update, _slasher_discount, _pack_attestations)}


def _call(eng, name, args, dev):
    """one call of b2_<name> (dev=False) or b2_<name>_dev: return code, outputs as numpy arrays, launches it made"""
    conv, outs, keep = [], [], []
    for a in args.values():
        if isinstance(a, DevOnly):
            if dev:
                conv.append(a.v)
        elif isinstance(a, Out):
            o = torch.full((a.n,), SENTINEL, dtype=torch.uint8, device="cuda") if dev else np.full(a.n, SENTINEL, np.uint8)
            outs.append(o)
            conv.append(o.data_ptr() if dev else o.ctypes.data)
        elif isinstance(a, In) and dev and not isinstance(a, HostIn):
            t = torch.from_numpy(np.frombuffer(a.a.tobytes(), np.uint8).copy()).cuda()
            keep.append(t)
            conv.append(t.data_ptr())
        elif isinstance(a, In):
            conv.append(a.a.ctypes.data)
        else:
            conv.append(a)
    if dev:
        conv.append(torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    before = eng.launch_count
    rc = getattr(eng.lib, "b2_" + name + ("_dev" if dev else ""))(eng.h, *conv)
    torch.cuda.synchronize()
    return rc, [o.cpu().numpy() if dev else o for o in outs], eng.launch_count - before


def _both_reject(eng, name, args):
    """both forms return B2_EINVAL with one message, launch nothing and write no output byte; returns the message"""
    from pos_evolution_b200._lib import B2_EINVAL
    texts = []
    for dev in (False, True):
        rc, outs, launches = _call(eng, name, args, dev)
        assert rc == B2_EINVAL, (name, dev)
        assert launches == 0, (name, dev)
        assert all((o == SENTINEL).all() for o in outs), (name, dev)
        texts.append(eng.lib.b2_last_error(eng.h).decode())
    assert texts[0] == texts[1], (name, texts)
    assert texts[0].startswith(name + ":"), texts[0]
    return texts[0]


def _load_state(eng, roots_seed=3):
    rng = np.random.default_rng(roots_seed)
    pks = eng.sk_to_pk(list(range(1, N_VAL + 1)))
    assert eng.registry_load(pks, rng.integers(16, 33, size=N_VAL).astype(np.uint64) * np.uint64(10**9)).all()
    parent, slot, roots, viable = scenarios.fork_tree(N_BLK, roots_seed)
    eng.tree_load(parent, slot, roots, viable)
    eng.latest_messages_load(rng.integers(0, 9, size=N_VAL).astype(np.uint64), rng.integers(0, N_BLK, size=N_VAL).astype(np.uint32),
                             (rng.random(N_VAL) < 0.8).astype(np.uint8), (rng.random(N_VAL) < 0.05).astype(np.uint8))
    for which in (0, 1):
        eng.participation_load(which, rng.integers(0, 8, size=N_VAL).astype(np.uint8))
    eng.sync_committee_load(pks[:16], 16)
    eng.slasher_init(N_VAL, 8, 4, EPOCH)
    return pks, roots


def _device_state(eng):
    return [*eng.latest_messages_read(), eng.participation_read(0), eng.participation_read(1), eng.get_weights(), eng.get_head(0), eng.equivocating()]


@pytest.fixture(scope="module")
def loaded():
    from pos_evolution_b200.engine import Engine
    eng = Engine(0)
    _, roots = _load_state(eng)
    yield eng, roots
    eng.close()


@pytest.mark.parametrize("name", list(PAIRS))
def test_both_forms_reject_alike(loaded, name):
    eng, roots = loaded
    args, bad, optional = PAIRS[name](eng, roots)
    for dev in (False, True):
        rc, _, _ = _call(eng, name, args, dev)
        assert rc == 0, (name, dev, eng.lib.b2_last_error(eng.h).decode())
    nulls = {"null " + k: {k: None} for k, v in args.items() if isinstance(v, (In, Out)) and k not in optional}
    for label, change in {**bad, **nulls}.items():
        state = _device_state(eng)
        _both_reject(eng, name, {**args, **change})
        for a, b in zip(state, _device_state(eng)):
            assert np.array_equal(a, b), (name, label)


# (pair, what the fresh engine holds, a substring of the message)
PRECONDITIONS = [
    ("fast_aggregate_verify", "", "registry not loaded"), ("aggregate_verify", "", "registry not loaded"),
    ("sync_aggregate_verify", "registry", "no sync committee loaded"), ("attestation_intake", "registry", "no tree loaded"),
    ("aggregate_and_proof_intake", "registry", "no tree loaded"), ("aggregate_and_proof_intake", "tree", "registry not loaded"),
    ("block_attestations", "", "registry not loaded"), ("block_attestations", "registry", "participation tables"),
    ("block_attestations_electra", "", "registry not loaded"), ("block_attestations_electra", "registry", "participation tables"),
    ("sync_committee_messages", "", "registry not loaded"), ("latest_messages_update", "", "registry not loaded"),
    ("slasher_advance", "registry", "b2_slasher_init"), ("slasher_update", "registry", "b2_slasher_init"),
    ("slasher_discount", "", "registry not loaded"), ("slasher_discount", "registry", "b2_slasher_init"),
    ("pack_attestations", "", "registry not loaded")]


@pytest.mark.parametrize("name,holds,why", PRECONDITIONS, ids=[f"{n}-{h or 'nothing'}" for n, h, _ in PRECONDITIONS])
def test_missing_state_is_rejected_alike(loaded, name, holds, why):
    from pos_evolution_b200.engine import Engine
    eng, roots = loaded
    args, _, _ = PAIRS[name](eng, roots)
    fresh = Engine(0)
    try:
        if holds == "registry":
            fresh.registry_load(eng.sk_to_pk(list(range(1, N_VAL + 1))), np.full(N_VAL, 32 * 10**9, np.uint64))
        elif holds == "tree":
            parent, slot, r, viable = scenarios.fork_tree(N_BLK, 3)
            fresh.tree_load(parent, slot, r, viable)
        assert why in _both_reject(fresh, name, args)
    finally:
        fresh.close()


@pytest.mark.parametrize("name", ["attestation_intake", "aggregate_and_proof_intake", "block_attestations", "block_attestations_electra"])
def test_device_form_refuses_n_sig_past_32_bits(loaded, name):
    """n_sig is the one count only the device form receives (the host form derives it from u32 offsets): 2^32 is refused, nothing
    launched, no output written"""
    from pos_evolution_b200._lib import B2_EINVAL
    eng, roots = loaded
    args, _, _ = PAIRS[name](eng, roots)
    state = _device_state(eng)
    rc, outs, launches = _call(eng, name, {**args, "n_sig": DevOnly(1 << 32)}, True)
    assert rc == B2_EINVAL and launches == 0 and all((o == SENTINEL).all() for o in outs)
    assert eng.lib.b2_last_error(eng.h).decode() == name + ": n_sig does not fit 32 bits"
    for a, b in zip(state, _device_state(eng)):
        assert np.array_equal(a, b)


def test_empty_shuffle_touches_nothing(loaded):
    """n_active = 0 returns at once through both forms: no launch, members_out untouched"""
    eng, roots = loaded
    args, _, _ = PAIRS["shuffle_committees"](eng, roots)
    for dev in (False, True):
        rc, outs, launches = _call(eng, "shuffle_committees", {**args, "n_active": 0}, dev)
        assert rc == 0 and launches == 0 and all((o == SENTINEL).all() for o in outs)
