"""tests/block_attestations_oracle.py against oracle.spec.process_attestation block by block on the MAINNET preset (CPU): 32-slot epochs,
so the source window is integer_squareroot(32) = 5 slots and the target window 32.  A small registry (512 validators: one committee of
16 per slot) keeps the spec's Python shuffle short.  Delays 1, 2, 5, 6, 31 and 32 into the previous table and 1, 2, 5, 6 and 31 into
the current one (a target-e attestation at delay 32 is included in epoch e + 1, where e is the previous epoch), delay 33, an attestation
of start(e - 1) at start(e) and one slot later, head and target mismatches at the window edges, order-exact credit across blocks, and a
fork at epoch e: previous-epoch attestations sign under the previous version.  The comparison is test_oracle_block_attestations.check."""
import copy
import hashlib

import pytest

import scenarios
from oracle import spec as S
from test_oracle_block_attestations import FakeBLS, Run, check, fake_sig

P = S.MAINNET
SPE = P.SLOTS_PER_EPOCH                  # 32; integer_squareroot = 5
E = 3
START = E * SPE                          # 96; e - 1 = slots 64-95
N_VAL = 512
KEYS = [hashlib.sha256(b"mainnet-pk" + i.to_bytes(4, "little")).digest() + bytes(16) for i in range(N_VAL)]
OLD, NEW = bytes.fromhex("00000001"), bytes.fromhex("00000002")


def _h(b):
    return hashlib.sha256(b).digest()


def make_run(slots, fork_epoch=0):
    """512 validators on the mainnet preset, the state at slots[0]; with fork_epoch, the fork from OLD to NEW at that epoch"""
    _, st = scenarios.minimal_state(N_VAL, slot=slots[0], preset=P, pks=KEYS)
    st.fork = S.Fork(OLD, NEW, fork_epoch) if fork_epoch else S.Fork(bytes(4), OLD, 0)
    st.previous_justified_checkpoint = S.Checkpoint(E - 2, _h(b"j-prev"))
    st.current_justified_checkpoint = S.Checkpoint(E - 1, _h(b"j-cur"))
    spec = S.Spec(P, bls_module=FakeBLS)
    assert spec.get_committee_count_per_slot(st, E) == 1 and len(spec.get_beacon_committee(st, START, 0)) == N_VAL // SPE
    return Run(spec, st, slots)


def test_mainnet_windows_and_masks():
    """block start(e): the previous table at delays 1, 2, 5, 6, 31, 32, a head mismatch at delay 1, target mismatches at delays 5 and 6;
    block start(e) + 31: the current table at delays 1, 2, 5, 6, 31 and the previous one at delay 32"""
    last = START + SPE - 1
    run = make_run((START, last))
    for d in (1, 2, 5, 6, 31, 32):
        run.add(0, START - d, 0)
    run.add(0, START - 1, 0, head=_h(b"other head"))
    run.add(0, START - 5, 0, target_root=_h(b"other target"))
    run.add(0, START - 6, 0, target_root=_h(b"other target"))
    for d in (1, 2, 5, 6, 31):
        run.add(1, last - d, 0)
    run.add(1, last - 32, 0)
    r = check(run)
    assert r["n_applied"] == 2 and r["status"].tolist() == [0] * 15
    assert r["flag_mask"].tolist() == [7, 3, 3, 2, 2, 2, 3, 1, 0] + [7, 3, 3, 2, 2, 2]
    assert r["numerator"][8] == 0 and r["numerator"][0] > 0


def test_mainnet_delay_33_and_the_first_slot_of_the_previous_epoch():
    """start(e - 1) is included at start(e) (delay 32) but not one slot later (delay 33, status 6), which stops the run at that block"""
    run = make_run((START, START + 1))
    run.add(0, START - SPE, 0)
    run.add(1, START, 0)
    assert check(run)["n_applied"] == 2
    run = make_run((START, START + 1, START + 2))
    run.add(0, START - 1, 0)
    run.add(1, START, 0)
    run.add(1, START - SPE, 0)
    run.add(2, START + 1, 0)
    r = check(run)
    assert r["status"].tolist() == [0, 0, 6, 0] and r["n_applied"] == 1 and r["block_status"].tolist() == [0, 1, 2]


def test_mainnet_order_exact_credit_across_blocks():
    """one committee of each epoch over four blocks: halves, then a superset, then an exact re-inclusion, with the delays crossing the
    source window; each later aggregate earns only the flags still unset"""
    run = make_run((START + 2, START + 4, START + 8, START + 20))
    half = [j < 8 for j in range(16)]
    run.add(0, START + 1, 0, bits=half)                              # delay 1: 7
    run.add(0, START - 3, 0, bits=[not b for b in half])            # delay 5: 3
    run.add(1, START + 1, 0, bits=[not b for b in half])            # delay 3: 3, the other half
    run.add(1, START - 3, 0)                                         # delay 7: 2, the first half's target only
    run.add(2, START + 1, 0)                                         # delay 7: 2, nothing left
    run.add(2, START - 3, 0)                                         # delay 11: nothing left
    run.add(3, START + 1, 0, bits=half)                              # delay 19: nothing left
    r = check(run)
    assert r["n_applied"] == 4 and r["flag_mask"].tolist() == [7, 3, 3, 2, 2, 2, 2]
    assert [int(x) > 0 for x in r["numerator"]] == [True, True, True, True, False, False, False]


def test_mainnet_fork_at_the_current_epoch():
    """state.fork.epoch == e: previous-epoch attestations sign under the previous version; one signed under the current version fails
    its signature check (status 11)"""
    run = make_run((START + 1, START + 3), fork_epoch=E)
    run.add(0, START, 0)
    run.add(0, START - 2, 0)
    run.add(1, START - 4, 0)
    assert check(run)["n_applied"] == 2
    sp, st = run.spec, run.state
    assert sp.get_domain(st, S.DOMAIN_BEACON_ATTESTER, E - 1) != sp.get_domain(st, S.DOMAIN_BEACON_ATTESTER, E)
    wrong = copy.copy(st)
    wrong.fork = S.Fork(NEW, NEW, 0)
    run.add(1, START - 5, 0)
    a = run.atts[1][-1]
    committee = sp.get_beacon_committee(st, a.data.slot, 0)
    a.signature = fake_sig([st.validators[v].pubkey for v in sorted(committee)],
                           sp.compute_signing_root(a.data, sp.get_domain(wrong, S.DOMAIN_BEACON_ATTESTER, E - 1)))
    r = check(run)
    assert r["status"].tolist() == [0, 0, 0, 11] and r["n_applied"] == 1


@pytest.mark.parametrize("bad", ["head", "target", "source"])
def test_mainnet_mismatches_at_the_window_edges(bad):
    """a head, target or source mismatch at delays 5 and 6 of the previous table: a head mismatch keeps source and target, a target
    mismatch keeps the source inside the window only, a source mismatch is status 9"""
    run = make_run((START + 4,))
    kw = {"head": dict(head=_h(b"h")), "target": dict(target_root=_h(b"t")),
          "source": dict(source=S.Checkpoint(E - 1, _h(b"j-cur")))}[bad]
    run.add(0, START - 1, 0, **kw)                                   # delay 5
    run.add(0, START - 2, 0, **kw)                                   # delay 6
    r = check(run)
    if bad == "source":
        assert r["status"].tolist() == [9, 9] and r["n_applied"] == 0 and r["block_first"][0] == 0
    else:
        assert r["flag_mask"].tolist() == ([3, 2] if bad == "head" else [1, 0]) and r["n_applied"] == 1
