"""Spec(incremental_tree=True): the decisions of the store mirror -- which tree calls it makes, with which block ids, and when it falls
back to a full upload -- checked on a stand-in engine whose answers come from oracle.fast over exactly the tables it was given, against
a brand-new Spec that re-uploads everything (so a stale or wrong tree shows up as a wrong head)."""
import numpy as np

from test_host_logic import _MirrorEngine, _mirror_world, _scratch_head, copy_state

DROP = 0xFFFFFFFF


class _TreeEngine(_MirrorEngine):
    """_MirrorEngine plus the in-place tree calls, applied to its host arrays as the device applies them"""

    def tree_load(self, parent, slot, roots, viable):
        super().tree_load(parent, slot, roots, viable)
        self.parent, self.viable = self.parent.astype(np.uint32), self.viable.astype(np.uint8)

    def tree_add(self, parent, slot, roots, viable):
        self.added = [int(p) for p in parent]
        self.parent = np.concatenate([self.parent, np.asarray(parent, dtype=np.uint32)])
        self.roots = np.vstack([self.roots, np.asarray(roots, dtype=np.uint8).reshape(-1, 32)])
        self.viable = np.concatenate([self.viable, np.asarray(viable, dtype=np.uint8)])
        self.log.append("tree_add")

    def tree_prune(self, r):
        n = len(self.parent)
        kept = np.zeros(n, dtype=bool)
        kept[r] = True
        for b in range(r + 1, n):
            kept[b] = kept[self.parent[b]]
        mp = np.full(n, DROP, dtype=np.uint32)
        mp[kept] = np.arange(int(kept.sum()), dtype=np.uint32)
        self.parent = mp[self.parent[kept]]
        self.parent[0] = 0
        self.roots, self.viable = self.roots[kept], self.viable[kept]
        old = self.m_block < n
        self.m_block[old] = mp[self.m_block[old]]
        self.log.append("tree_prune")
        return mp

    def tree_set_viable(self, idx, viable):
        self.viable[np.asarray(idx, dtype=np.int64)] = viable
        self.log.append("tree_set_viable")

    def get_weights(self, boost_idx, boost_score):
        from oracle import fast
        has = self.m_has * (self.m_block < len(self.parent))
        return fast.ghost_weights(self.parent, np.where(has != 0, self.m_block, 0), has, self.eff, self.flags & 1, self.equiv, boost_idx, boost_score)


def _vote(PS, sp, store, root, validators, epoch):
    att = PS.Attestation([True] * len(validators), PS.AttestationData(8, 0, root, PS.Checkpoint(0, root), PS.Checkpoint(epoch, root)), bytes(96))
    sp.update_latest_messages(store, validators, att)


def _add(PS, store, root, parent_root, state_of):
    store.blocks[root] = PS.BeaconBlock(store.blocks[parent_root].slot + 1, parent_root)
    store.block_states[root] = state_of


def test_incremental_mirror_decisions():
    from pos_evolution_b200 import spec as PS
    eng = _TreeEngine()
    sp = PS.Spec(PS.MINIMAL, engine=eng, incremental_tree=True)
    store, state, rb, slot = _mirror_world(PS)
    assert sp.get_head(store) == _scratch_head(PS, store)
    assert eng.log == ["registry_load", "balances", "tree_load", "lmd_load"]
    leaf_state = store.block_states[rb[7]]
    # a new block: one tree_add under its parent's id, no upload
    eng.log.clear()
    _add(PS, store, b"\x41" * 32, rb[7], leaf_state)
    assert sp.get_head(store) == _scratch_head(PS, store)
    assert eng.log == ["tree_add"] and eng.added == [sp._mirror["index"][rb[7]]] and sp._mirror["index"][b"\x41" * 32] == 40
    # a batch with a fork inside it, then a vote for the newest block before any get_head: appended first, then the vote
    eng.log.clear()
    _add(PS, store, b"\x42" * 32, b"\x41" * 32, leaf_state)
    _add(PS, store, b"\x43" * 32, b"\x41" * 32, leaf_state)
    _add(PS, store, b"\x44" * 32, b"\x43" * 32, leaf_state)
    _vote(PS, sp, store, b"\x44" * 32, list(range(30)), 5)
    assert eng.log == ["tree_add", "lmd_update"] and eng.added == [40, 40, 42]
    assert sp.get_head(store) == _scratch_head(PS, store) == b"\x44" * 32
    assert eng.log == ["tree_add", "lmd_update"]
    # justification and finalization move down the chain to block 0x41: one prune, the leaves' bytes follow the new checkpoints
    eng.log.clear()
    J, F = PS.Checkpoint(2, b"\x43" * 32), PS.Checkpoint(2, b"\x41" * 32)
    viable_state = copy_state(PS, leaf_state)
    viable_state.current_justified_checkpoint, viable_state.finalized_checkpoint = J, F
    store.block_states[b"\x42" * 32] = viable_state
    store.justified_checkpoint, store.finalized_checkpoint = J, F
    store.checkpoint_states[J] = state
    assert sp.get_head(store) == _scratch_head(PS, store)
    assert eng.log == ["tree_prune", "tree_set_viable"] and sp.stats["tree_prunes"] == 1 and sp.stats["viability_updates"] == 1
    assert sp._mirror["order"] == [b"\x41" * 32, b"\x42" * 32, b"\x43" * 32, b"\x44" * 32] and len(eng.parent) == 4
    assert sp.stats["store_uploads"] == 1 and sp.stats["tree_adds"] == 2
    # the vote table was re-mapped, not re-uploaded: validators 0..29 still vote for 0x44, now id 3
    assert (eng.m_block[:30] == 3).all()
    # a block outside the finalized subtree is not mirrored; a vote for it falls back to a full upload
    eng.log.clear()
    _add(PS, store, b"\x45" * 32, rb[3], leaf_state)
    assert sp.get_head(store) == _scratch_head(PS, store) and eng.log == []
    _vote(PS, sp, store, b"\x45" * 32, [40], 6)
    assert sp.get_head(store) == _scratch_head(PS, store) and "tree_load" in eng.log and sp.stats["store_uploads"] == 2
    # a finalized block the tree does not hold: full upload
    eng.log.clear()
    store.finalized_checkpoint = PS.Checkpoint(2, rb[3])
    store.block_states[b"\x42" * 32].finalized_checkpoint = store.finalized_checkpoint
    assert sp.get_head(store) == _scratch_head(PS, store) and "tree_load" in eng.log


def test_default_spec_keeps_reloading():
    """without incremental_tree a new block still re-uploads the store, as before"""
    from pos_evolution_b200 import spec as PS
    eng = _TreeEngine()
    sp = PS.Spec(PS.MINIMAL, engine=eng)
    store, state, rb, slot = _mirror_world(PS)
    sp.get_head(store)
    eng.log.clear()
    _add(PS, store, b"\x41" * 32, rb[7], store.block_states[rb[7]])
    assert sp.get_head(store) == _scratch_head(PS, store) and eng.log == ["tree_load", "lmd_load"]
