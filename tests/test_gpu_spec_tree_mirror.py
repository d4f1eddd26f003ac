"""Spec(incremental_tree=True) on the GPU: a store grown slot by slot, with forks, votes and justification / finalization moving, keeps
its device tree current by tree_add / tree_prune / tree_set_viable after one upload, and every head equals the one a brand-new Spec
computes from scratch over the oracle stand-in engine."""
import numpy as np
import pytest

from test_host_logic import _MirrorEngine, _mirror_world, _scratch_head, copy_state

gpu = pytest.mark.gpu


@gpu
def test_store_grown_slot_by_slot():
    from pos_evolution_b200 import spec as PS
    from pos_evolution_b200.engine import Engine
    rng = np.random.default_rng(9)
    sp = PS.Spec(PS.MINIMAL, engine=Engine(0), incremental_tree=True)
    store, state, rb, slot = _mirror_world(PS)
    n_val = len(state.validators)
    base = store.block_states[rb[0]]
    assert sp.get_head(store) == _scratch_head(PS, store)
    chain, epoch = [sp.get_head(store)], 2
    for s in range(1, 49):
        bs = copy_state(PS, base)
        bs.current_justified_checkpoint, bs.finalized_checkpoint = store.justified_checkpoint, store.finalized_checkpoint
        parent = chain[-1] if s % 5 else chain[max(0, len(chain) - 3)]           # every fifth block forks off an older chain block
        root = (0x1000 + s).to_bytes(2, "big") * 16
        store.blocks[root] = PS.BeaconBlock(store.blocks[parent].slot + 1, parent)
        store.block_states[root] = bs
        if s % 5:
            chain.append(root)
        voters = sorted(int(v) for v in rng.choice(n_val, 12, replace=False))
        att = PS.Attestation([True] * len(voters), PS.AttestationData(8, 0, root, PS.Checkpoint(0, root), PS.Checkpoint(epoch, root)), bytes(96))
        sp.update_latest_messages(store, voters, att)
        epoch += 1
        if s % 8 == 0 and len(chain) > 3:                                        # justification and finalization move down the chain
            J = PS.Checkpoint(epoch, chain[-2])
            store.finalized_checkpoint = PS.Checkpoint(epoch, store.justified_checkpoint.root)
            store.justified_checkpoint = J
            store.checkpoint_states[J] = state
            bs.current_justified_checkpoint, bs.finalized_checkpoint = store.justified_checkpoint, store.finalized_checkpoint
        if s % 3 == 0:
            store.proposer_boost_root = chain[-1]
        assert sp.get_head(store) == _scratch_head(PS, store), s
        for r in (store.justified_checkpoint.root, chain[-1]):
            assert sp.get_weight(store, r) == PS.Spec(PS.MINIMAL, engine=_MirrorEngine()).get_weight(store, r)
    assert sp.stats["store_uploads"] == 1
    assert sp.stats["tree_adds"] >= 40 and sp.stats["tree_prunes"] >= 4 and sp.stats["viability_updates"] >= 1
