"""CPU check of tests/votes_oracle.py, the model of b2_votes_group_dev the GPU tests compare against: its outputs against a
position-by-position restatement of the layout (include/b200pos.h) on small ragged committees."""
import numpy as np
import pytest

import votes_oracle as VO


@pytest.mark.parametrize("seed", range(4))
def test_group_outputs_equal_a_per_position_restatement(seed):
    rng = np.random.default_rng(seed)
    sizes = rng.integers(1, 17, size=7)
    off = np.concatenate([[0], np.cumsum(sizes)])
    nv = rng.integers(1, 5, size=7)
    vote_off = np.concatenate([[0], np.cumsum(nv)])
    vote = np.full(int(off[-1]), VO.NONE, dtype=np.int64)
    for c in range(7):
        vote[off[c]:off[c + 1]] = np.where(rng.random(sizes[c]) < 0.2, VO.NONE, vote_off[c] + rng.integers(0, nv[c], size=sizes[c]))
    vote[off[2]] = vote_off[5]                                         # another committee's id: not attesting
    members = rng.permutation(int(off[-1])).astype(np.uint32)
    sigs = rng.integers(0, 256, size=(int(off[-1]), 96), dtype=np.uint8)
    c0, c1 = 2, 6
    g = VO.group_outputs(members, off, vote, vote_off, sigs[off[c0]:off[c1]], 2, c0, c1)
    members_out, pos_out, seg = [], [], []
    bits, agg = np.zeros((int(vote_off[-1]), 2), np.uint8), np.zeros((int(vote_off[-1]), 2), np.uint8)
    sigs_out = []
    for c in range(7):
        v0, v1 = int(vote_off[c]), int(vote_off[c + 1])
        att = lambda j: v0 <= vote[off[c] + j] < v1      # noqa: E731
        for v in range(v0, v1):
            seg.append(len(pos_out))
            pos = [j for j in range(sizes[c]) if att(j) and vote[off[c] + j] == v] + ([j for j in range(sizes[c]) if not att(j)] if v == v1 - 1 else [])
            for i, j in enumerate(pos):
                members_out.append(members[off[c] + j])
                pos_out.append(j)
                if att(j):
                    bits[v, i >> 3] |= 1 << (i & 7)
                    agg[v, j >> 3] |= 1 << (j & 7)
                if c0 <= c < c1:
                    sigs_out.append(sigs[off[c] + j] if att(j) else VO.INFINITY96)
    seg.append(len(pos_out))
    assert g.members_out.tolist() == [int(x) for x in members_out] and g.pos_out.tolist() == pos_out and g.seg_off.tolist() == seg
    assert g.seg_off_loc.tolist() == [s - int(off[c0]) for s in seg[vote_off[c0]:vote_off[c1] + 1]]
    assert np.array_equal(g.bits, bits) and np.array_equal(g.agg_bits, agg) and np.array_equal(g.sigs_out, np.array(sigs_out))
